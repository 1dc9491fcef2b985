"""BiLSTM training (csrc/lstm.cu forward_train, csrc/lstm_bwd.cu) and the wgmma inference forward (csrc/lstm_umma.cu) at
the shapes that train and rank, against the float64 oracle (oracle/lstm_bwd_ref.py, evaluated 128 sequences at a time)
(needs an H100 except the workspace sweep).

The backward's weight-gradient reduction splits the batch into at most MAX_CHUNKS = 32 chunks of whole sequences and its
recurrence runs 8 sequences per CTA, so the batch sizes below are chosen against both: 512 (the stream batch, 32 x 16),
1000 (32 x 32, last chunk 8), 4095 (32 x 128, last chunk 127, last CTA 7), 257 (29 x 9).  The wgmma forward runs
G = (SMs / 8) & ~1 groups, each covering one 64-sequence tile per direction and slot per round, so B = 64 G + 1 puts one
sequence in a second round.  Gradients are held to the bound of tests/test_gpu_lstm_train.py,
|got - want| <= 2e-4 |want| + 2e-5 rms(want), widened only as far as fp32 CPU torch.nn.LSTM autograd lands on the same case;
the worst error ratio against that bound is printed per tensor, with the oracle's wall time."""
import ctypes as C
import time

import numpy as np
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence

from nerrf_b200 import _lib as L
from nerrf_b200.ai import autograd as AG
from nerrf_b200.ai.models.lstm import LSTMScorer
from oracle import lstm_bwd_ref as LB

RTOL, ATOL_RMS = 2e-4, 2e-5
H, MAX_CHUNKS, BS = 256, 32, 8
SLICE = 128                       # sequences per float64 oracle pass
gpu = pytest.mark.gpu


def _plan(B):
    """(sequences per chunk, chunks) of the weight-gradient reduction: a function of B alone."""
    c = min(B, MAX_CHUNKS) if B > 0 else 1
    spc = max(1, -(-B // c))
    return spc, max(1, -(-B // spc))


def _sizes(B, T, D_in, layers):
    """(tape bytes, workspace bytes) restated from lstm_tape.cuh and bwd_plan."""
    up = lambda x: (x + 255) & ~255
    _, chunks = _plan(B)
    nmax = max(D_in, H, 2 * H if layers > 1 else 0)
    tape = layers * B * T * (2 * H + 2 * 4 * H + 2 * H) * 4
    return tape, up(B * T * 2 * H * 4) + up(2 * chunks * 4 * H * nmax * 4) + 2 * chunks * 4 * H * 4


def _ratio(got, want):
    """max |got - want| / (RTOL |want| + ATOL_RMS rms(want)): <= 1 is inside the bound."""
    got = np.asarray(got.detach().double().cpu().numpy() if hasattr(got, "detach") else got, np.float64)
    want = np.asarray(want, np.float64)
    assert got.shape == want.shape
    assert np.isfinite(got).all()
    if want.size == 0:
        return 0.0
    rms = float(np.sqrt((want ** 2).mean()))
    return float((np.abs(got - want) / (RTOL * np.abs(want) + ATOL_RMS * max(rms, 1e-30))).max())


def _lengths(B, T, g, lo=0):
    """Uniform in [lo, T], with 0, 1 and T at both ends of the batch (the last sequence full length)."""
    ln = torch.randint(lo, T + 1, (B,), generator=g)
    for i, v in ((0, T), (1, 0), (2, 1), (-3, 1), (-2, 0), (-1, T)):
        if B > 5:
            ln[i] = v
    return ln


def _batch(B, T, D, seed, lo=0):
    """seq random everywhere, padded tails included (they must not be read)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, T, D, generator=g), _lengths(B, T, g, lo), torch.randn(B, 2, generator=g)


def _lstm_names(L_):
    return [f"lstm.{n}_l{l}{sfx}" for l in range(L_) for sfx in ("", "_reverse")
            for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]


def _names(L_):
    return _lstm_names(L_) + ["head.weight", "head.bias"]


def _flat_oracle(w, L_, head=True):
    flat = [g for layer in w["lstm"] for d in layer for g in d]
    names = _lstm_names(L_)
    if head:
        flat += [w["head_W"], w["head_b"]]
        names = _names(L_)
    return dict(zip(names, flat))


def _torch_fp32(scorer, seq, lengths, dlogit=None, dhfin=None):
    """fp32 CPU torch.nn.LSTM autograd of the same case (the witness a widened bound must cite): gradients of
    sum(dlogit * logits) or of sum(dhfin * hfin).  pack_padded_sequence refuses zero-length sequences: they are left out,
    and their exact contribution (dlogit to the head bias, nothing else) is added back."""
    cpu = LSTMScorer(scorer.in_dim, H, scorer.num_layers, seed=None)
    cpu.load_state_dict({k: v.detach().cpu() for k, v in scorer.state_dict().items()})
    T = seq.shape[1]
    keep = lengths > 0
    x = seq[keep].clone().requires_grad_()
    packed = pack_padded_sequence(x, lengths[keep].clamp(max=T), batch_first=True, enforce_sorted=False)
    _, (hn, _) = cpu.lstm(packed)
    feat = torch.cat([hn[-2], hn[-1]], 1)
    if dlogit is not None:
        (cpu.head(feat) * dlogit[keep]).sum().backward()
    else:
        (feat * dhfin[keep]).sum().backward()
    params = dict(cpu.named_parameters())
    grads = {n: params[n].grad.clone() for n in _names(cpu.num_layers) if params[n].grad is not None}
    if dlogit is not None:
        grads["head.bias"] += dlogit[~keep].sum(0)
    dseq = torch.zeros_like(seq)
    dseq[keep] = x.grad
    grads["dseq"] = dseq
    return grads


def _check(got, want, witness, what):
    """Every tensor of `got` within the bound of `want`; the fp32 torch witness is computed only if some tensor is not."""
    ratios = {k: _ratio(got[k], want[k]) for k in got}
    allowed = {k: 1.0 for k in got}
    if max(ratios.values()) > 1.0:
        ref = witness()
        allowed = {k: max(1.0, _ratio(ref[k], want[k])) if k in ref else 1.0 for k in got}
    print(f"{what}: " + ", ".join(f"{k} {r:.3f}" + (f" (torch {allowed[k]:.3f})" if allowed[k] > 1 else "")
                                  for k, r in ratios.items()))
    for k, r in ratios.items():
        assert r <= allowed[k], f"{what} {k}: error ratio {r:.3f} > {allowed[k]:.3f}"
    return ratios


def _timed(what, fn, *a, **k):
    t = time.perf_counter()
    out = fn(*a, **k)
    print(f"{what}: float64 oracle {time.perf_counter() - t:.1f} s")
    return out


# --------------------------------------------------------------------------------------------- the C ABI, directly
def _weights(scorer):
    """(W_ih, W_hh) in torch layout for the backward, (W_ih^T, W_hh^T, b_ih + b_hh) for the forward, as LSTMFn builds them."""
    p = [w.detach() for w in AG.lstm_params(scorer)]
    n = 2 * scorer.num_layers
    W_ih = [p[4 * i].contiguous() for i in range(n)]
    W_hh = [p[4 * i + 1].contiguous() for i in range(n)]
    return W_ih, W_hh, [w.t().contiguous() for w in W_ih], [w.t().contiguous() for w in W_hh], \
        [(p[4 * i + 2] + p[4 * i + 3]).contiguous() for i in range(n)]


def _need(B, T, D, layers, H_=H):
    tb, wb = C.c_size_t(), C.c_size_t()
    L.check(L.lib().nerrf_lstm_train_workspace_bytes(B, T, D, H_, layers, C.byref(tb), C.byref(wb)), "workspace_bytes")
    return tb.value, wb.value


def _fwd(scorer, seq, ln, tape, tape_bytes=None, H_=H, tape_ptr=None, B=None):
    """One nerrf_lstm_forward_train call -> (rc, hfin).  B overrides seq.shape[0] (torch gives an empty tensor a null
    pointer, so a B = 0 call passes a one-row buffer)."""
    B = seq.shape[0] if B is None else B
    T, D = seq.shape[1:]
    _, _, wih_t, whh_t, bias = _weights(scorer)
    hfin = torch.empty(max(B, 1), 2 * H, device="cuda")             # a live pointer even when B = 0
    rc = L.lib().nerrf_lstm_forward_train(L.ptr(seq), L.ptr(ln), B, T, D, H_, scorer.num_layers, L.ptr_array(wih_t),
                                          L.ptr_array(whh_t), L.ptr_array(bias), L.ptr(hfin),
                                          tape_ptr or L.ptr(tape), tape.numel() if tape_bytes is None else tape_bytes,
                                          L.current_stream_ptr())
    torch.cuda.synchronize()
    return rc, hfin[:B]


def _bwd(scorer, seq, ln, tape, dhfin, ws, dseq=True, tape_bytes=None, ws_bytes=None, H_=H, tape_ptr=None, ws_ptr=None,
         fill=None, B=None):
    """One nerrf_lstm_backward call -> (rc, grads dict with dseq unless dseq=False).  fill: initial value of the outputs."""
    B = seq.shape[0] if B is None else B
    T, D = seq.shape[1:]
    W_ih, W_hh, _, _, _ = _weights(scorer)
    mk = (lambda like: torch.full_like(like, fill)) if fill is not None else torch.empty_like
    dW_ih, dW_hh = [mk(w) for w in W_ih], [mk(w) for w in W_hh]
    db = [mk(torch.empty(4 * H, device="cuda")) for _ in W_ih]
    out_seq = mk(seq) if dseq else None
    rc = L.lib().nerrf_lstm_backward(L.ptr(seq), L.ptr(ln), B, T, D, H_, scorer.num_layers, L.ptr_array(W_ih),
                                     L.ptr_array(W_hh), tape_ptr or L.ptr(tape),
                                     tape.numel() if tape_bytes is None else tape_bytes, L.ptr(dhfin), L.ptr(out_seq),
                                     L.ptr_array(dW_ih), L.ptr_array(dW_hh), L.ptr_array(db), ws_ptr or L.ptr(ws),
                                     ws.numel() if ws_bytes is None else ws_bytes, L.current_stream_ptr())
    torch.cuda.synchronize()
    names = _lstm_names(scorer.num_layers)
    got = {}
    for i in range(len(W_ih)):
        got[names[4 * i]], got[names[4 * i + 1]], got[names[4 * i + 2]] = dW_ih[i], dW_hh[i], db[i]
    if dseq:
        got["dseq"] = out_seq
    return rc, got


def _buffers(B, T, D, layers):
    tb, wb = _need(B, T, D, layers)
    return torch.empty(tb, dtype=torch.uint8, device="cuda"), torch.empty(wb, dtype=torch.uint8, device="cuda")


def _abi_round(scorer, seq, ln, dhfin, tape, ws, dseq=True):
    rc, hfin = _fwd(scorer, seq, ln, tape)
    L.check(rc, "nerrf_lstm_forward_train")
    rc, got = _bwd(scorer, seq, ln, tape, dhfin, ws, dseq=dseq)
    L.check(rc, "nerrf_lstm_backward")
    return hfin, got


ABI_CASES = [  # B, T, layers, D_in, lower bound of the ragged lengths
    (512, 100, 2, 16, 0),
    (1000, 100, 2, 16, 0),
    (4095, 100, 2, 16, 50),
    (257, 30, 3, 5, 0),
    (2048, 1, 2, 16, 0),
    (600, 100, 2, 64, 0),
]


@gpu
@pytest.mark.parametrize("B,T,layers,D,lo", ABI_CASES)
def test_backward_through_the_abi_at_scale(B, T, layers, D, lo):
    """forward_train + backward with a random dhfin, against the float64 statement of sum(dhfin * hfin) (the oracle with
    an identity head).  hfin is checked too.  A second call gives the same bits, and a call with dseq = NULL gives the
    weight-gradient bits of the full call."""
    scorer = LSTMScorer(D, H, layers, seed=B + T).cuda()
    seq, lengths, _ = _batch(B, T, D, seed=B * 7 + T + layers, lo=lo)
    dhfin = torch.randn(B, 2 * H, generator=torch.Generator().manual_seed(B + 1))
    s, ln, dh = seq.cuda(), lengths.to(torch.int32).cuda(), dhfin.cuda()
    tape, ws = _buffers(B, T, D, layers)
    hfin, got = _abi_round(scorer, s, ln, dh, tape, ws)

    P = scorer.oracle_params()
    P["head_W"], P["head_b"] = np.eye(2 * H), np.zeros(2 * H)
    w = _timed(f"B={B} T={T}", LB.model_backward, P, seq, lengths, dhfin, batch=SLICE)
    want = _flat_oracle(w, layers, head=False)
    want["dseq"] = w["seq"]
    want_h = w["logits"]                                            # hfin, through the identity head
    spc, chunks = _plan(B)
    what = (f"B={B} T={T} L={layers} D={D} ({chunks} chunks x {spc} seqs, last {B - (chunks - 1) * spc}; "
            f"last CTA {B - (B - 1) // BS * BS}) hfin {_ratio(hfin, want_h):.3f}")
    assert _ratio(hfin, want_h) <= 1.0, "hfin"
    _check(got, want, lambda: _torch_fp32(scorer, seq, lengths, dhfin=dhfin), what)

    hfin2, again = _abi_round(scorer, s, ln, dh, tape, ws)
    assert torch.equal(hfin, hfin2)
    for k in got:
        assert torch.equal(got[k], again[k]), f"second call: {k}"
    _, no_dseq = _abi_round(scorer, s, ln, dh, tape, ws, dseq=False)
    assert "dseq" not in no_dseq
    for k in no_dseq:
        assert torch.equal(got[k], no_dseq[k]), f"dseq = NULL: {k}"


# ------------------------------------------------------------------------------------------- stream-window sequences
def _probs_all_paths(scorer, seq, ln, monkeypatch):
    """(wgmma inference, fp32 CUDA-core inference, sigmoid of forward_train's logits) probabilities."""
    out = []
    for algo in ("umma", "ffma"):
        monkeypatch.setenv("NERRF_LSTM_ALGO", algo)
        out.append(scorer(seq, ln).cpu().double())
    monkeypatch.delenv("NERRF_LSTM_ALGO")
    with torch.no_grad():
        out.append(torch.sigmoid(AG.lstm_logits(scorer, seq, ln)).cpu().double())
    return out


def _check_probs(probs, want, what):
    errs = [float((p - want).abs().max()) for p in probs]
    print(f"{what}: max |prob - fp64| wgmma {errs[0]:.2e}, ffma {errs[1]:.2e}, forward_train {errs[2]:.2e}")
    for name, e in zip(("wgmma", "ffma", "forward_train"), errs):
        assert e < 1e-5, f"{what}: {name} probabilities off by {e:.2e}"


@gpu
def test_stream_window_sequences(monkeypatch):
    """Sequences built on the device from fleet windows (one-hot slots plus small ramps, most truncated to T = 100):
    every LSTMScorer gradient and dseq under the training loss of ai.train.train, and the probabilities of both inference
    paths and of forward_train."""
    from nerrf_b200 import stream
    from nerrf_b200.ai import train as TR
    cols, _ = stream.fleet_columns(1500, 10, seed=0, bystanders=2)
    exs = TR.stream_examples(cols, 2, seed=0, files_per_window=512)
    bce = torch.nn.functional.binary_cross_entropy_with_logits
    for k, ex in enumerate(exs):
        seq, ln, y = ex["seq"], ex["lengths"], ex["seq_label"]
        B, T, D = seq.shape
        lens = ln.cpu().numpy()
        hist = np.histogram(lens, bins=[0, 1, 2, 11, 26, 51, 76, T, T + 1])[0]
        print(f"window {k} {ex['window']}: B={B} T={T}, {int((lens == T).sum())} truncated to T; lengths "
              f"[0 | 1 | 2-10 | 11-25 | 26-50 | 51-75 | 76-{T - 1} | {T}] = {hist.tolist()}")
        assert B > 256
        scorer = LSTMScorer(D, H, 2, seed=40 + k).cuda()
        scorer.zero_grad(set_to_none=True)
        x = seq.detach().clone().requires_grad_()
        sl = AG.lstm_logits(scorer, x, ln)
        sl.retain_grad()
        (bce(sl[:, 0], y) + 0.5 * bce(sl[:, 1], y)).backward()       # the LSTM term of ai.train.train's loss
        dlogit = sl.grad.detach().cpu()
        params = dict(scorer.named_parameters())
        got = {n: params[n].grad for n in _names(2)}
        got["dseq"] = x.grad
        seq_c, ln_c = seq.cpu(), ln.cpu()
        P = scorer.oracle_params()
        w = _timed(f"window {k}", LB.model_backward, P, seq_c, ln_c, dlogit, batch=SLICE)
        want = _flat_oracle(w, 2)
        want["dseq"] = w["seq"]
        _check(got, want, lambda: _torch_fp32(scorer, seq_c, ln_c.long(), dlogit=dlogit), f"window {k} gradients")
        want_p = torch.sigmoid(torch.from_numpy(w["logits"]))
        _check_probs(_probs_all_paths(scorer, seq, ln, monkeypatch), want_p, f"window {k}")


# ------------------------------------------------------------------------------------------------------ saturation
@gpu
@pytest.mark.parametrize("scale", [30, 300])
def test_saturated_gates(scale, monkeypatch):
    """Inputs x30 and x300: first-layer gate pre-activations of tens to hundreds, where expf overflows and 1 - i cancels
    (the fraction of saturated gates is printed).  No NaN or inf, every gradient within the bound (at x300 a few tensors
    need the fp32 torch witness's widening), probabilities on every path within 1e-5."""
    B, T, D = 300, 100, 16
    scorer = LSTMScorer(D, H, 2, seed=21).cuda()
    seq, lengths, dlogit = _batch(B, T, D, seed=21)
    seq = seq * scale
    P = scorer.oracle_params()
    fw = [LB._arr(w, np.float64) for w in P["lstm"][0][0]]
    _, _, tp = LB.direction_forward(seq[:32].double().numpy(), lengths[:32].numpy(), *fw, reverse=False)
    gates = tp["gates"][np.arange(T)[None, :] < lengths[:32].numpy()[:, None]]
    sat = float(np.mean(np.minimum(np.abs(gates), 1 - np.abs(gates)) < 1e-3))
    print(f"x{scale}: {sat:.2f} of layer-0 forward gates within 1e-3 of 0 or +-1")
    s, ln = seq.cuda(), lengths.cuda()
    scorer.zero_grad(set_to_none=True)
    x = s.clone().requires_grad_()
    (AG.lstm_logits(scorer, x, ln) * dlogit.cuda()).sum().backward()
    params = dict(scorer.named_parameters())
    got = {n: params[n].grad for n in _names(2)}
    got["dseq"] = x.grad
    for k, v in got.items():
        assert torch.isfinite(v).all(), k
    w = _timed(f"x{scale}", LB.model_backward, P, seq, lengths, dlogit, batch=SLICE)
    want = _flat_oracle(w, 2)
    want["dseq"] = w["seq"]
    _check(got, want, lambda: _torch_fp32(scorer, seq, lengths, dlogit=dlogit), f"x{scale} gradients")
    want_p = torch.sigmoid(torch.from_numpy(w["logits"]))
    probs = _probs_all_paths(scorer, s, ln, monkeypatch)
    for p in probs:
        assert torch.isfinite(p).all()
    _check_probs(probs, want_p, f"x{scale}")


# ------------------------------------------------------------------------------------------ every row of the wgmma path
def _groups():
    """G of lstm_umma.cu's groups_for_device: recurrence groups of 8 CTAs, an even number, one CTA per SM."""
    g = (torch.cuda.get_device_properties(0).multi_processor_count // 8) & ~1
    return g if g >= 2 else 0


UMMA_CASES = [  # id, B as a function of G, layers, D_in
    ("64G", lambda G: 64 * G, 2, 16),
    ("64G+1", lambda G: 64 * G + 1, 2, 16),
    ("128G-1", lambda G: 128 * G - 1, 2, 16),
    ("4096", lambda G: 4096, 2, 16),
    ("64G+1 3 layers", lambda G: 64 * G + 1, 3, 16),
    ("64G+33 D64", lambda G: 64 * G + 33, 2, 64),
]


@gpu
@pytest.mark.parametrize("case", UMMA_CASES, ids=[c[0] for c in UMMA_CASES])
def test_wgmma_forward_every_row(case, monkeypatch):
    """Every row of the wgmma forward against the float64 logits (< 1e-5 in probability, the check of
    tests/test_gpu_lstm.py) and against the fp32 CUDA-core kernel (< 2e-6), at batch sizes that end a round exactly,
    leave one sequence or a partial tile in a later round, or run four rounds."""
    name, fB, layers, D = case
    G = _groups()
    B, T = fB(G), 100
    n_bt = -(-B // 64)
    scorer = LSTMScorer(D, H, layers, seed=B + layers).cuda()
    seq, lengths, _ = _batch(B, T, D, seed=B * 3 + D + layers)
    s, ln = seq.cuda(), lengths.cuda()
    monkeypatch.setenv("NERRF_LSTM_ALGO", "umma")
    got = scorer(s, ln).cpu().double()
    monkeypatch.setenv("NERRF_LSTM_ALGO", "ffma")
    ref = scorer(s, ln).cpu().double()
    want = torch.sigmoid(torch.from_numpy(_timed(f"{name} (B={B})", LB.logits, scorer.oracle_params(), seq, lengths,
                                                 batch=SLICE)))
    e_w, e_f, e_x = (float((got - want).abs().max()), float((ref - want).abs().max()), float((got - ref).abs().max()))
    print(f"{name}: G={G} B={B} ({n_bt} tiles per direction, {-(-n_bt // G)} rounds) L={layers} D={D}: max |prob - fp64| "
          f"wgmma {e_w:.2e}, ffma {e_f:.2e}; wgmma - ffma {e_x:.2e}")
    assert e_w < 1e-5 and e_f < 1e-5
    assert e_x < 2e-6


# ----------------------------------------------------------------------------------------------------------- ABI edges
@gpu
def test_empty_batch_zeroes_the_gradients():
    scorer = LSTMScorer(16, H, 2, seed=1).cuda()
    seq = torch.zeros(1, 10, 16, device="cuda")                    # live pointers; B = 0 reads none of them
    ln = torch.zeros(1, dtype=torch.int32, device="cuda")
    tb, wb = _need(0, 10, 16, 2)
    assert (tb, wb) == _sizes(0, 10, 16, 2) and tb == 0
    tape = torch.empty(16, dtype=torch.uint8, device="cuda")
    ws = torch.empty(wb, dtype=torch.uint8, device="cuda")
    rc, _ = _fwd(scorer, seq, ln, tape, B=0)
    assert rc == 0, L.lib().nerrf_last_error()
    rc, got = _bwd(scorer, seq, ln, tape, torch.zeros(1, 2 * H, device="cuda"), ws, dseq=False, fill=float("nan"), B=0)
    assert rc == 0, L.lib().nerrf_last_error()
    assert len(got) == 12
    for k, v in got.items():
        assert v.numel() and int(torch.count_nonzero(v)) == 0, k


@gpu
def test_short_misaligned_and_wrong_width_buffers_are_refused():
    B, T, D = 37, 20, 16
    scorer = LSTMScorer(D, H, 2, seed=2).cuda()
    seq, lengths, _ = _batch(B, T, D, seed=2)
    s, ln = seq.cuda(), lengths.to(torch.int32).cuda()
    dh = torch.randn(B, 2 * H, device="cuda")
    tb, wb = _need(B, T, D, 2)
    assert (tb, wb) == _sizes(B, T, D, 2)
    tape = torch.empty(tb + 16, dtype=torch.uint8, device="cuda")
    ws = torch.empty(wb + 16, dtype=torch.uint8, device="cuda")
    lib = L.lib()
    assert _fwd(scorer, s, ln, tape, tape_bytes=tb - 1)[0] == -4 and b"tape too small" in lib.nerrf_last_error()
    L.check(_fwd(scorer, s, ln, tape, tape_bytes=tb)[0])
    assert _bwd(scorer, s, ln, tape, dh, ws, tape_bytes=tb - 1, ws_bytes=wb)[0] == -4
    assert b"tape too small" in lib.nerrf_last_error()
    assert _bwd(scorer, s, ln, tape, dh, ws, tape_bytes=tb, ws_bytes=wb - 1)[0] == -4
    assert b"workspace too small" in lib.nerrf_last_error()
    off = lambda t: C.c_void_p(t.data_ptr() + 4)
    assert _fwd(scorer, s, ln, tape, tape_bytes=tb, tape_ptr=off(tape))[0] == -1
    assert b"16-byte aligned" in lib.nerrf_last_error()
    assert _bwd(scorer, s, ln, tape, dh, ws, tape_bytes=tb, ws_bytes=wb, tape_ptr=off(tape))[0] == -1
    assert b"16-byte aligned" in lib.nerrf_last_error()
    assert _bwd(scorer, s, ln, tape, dh, ws, tape_bytes=tb, ws_bytes=wb, ws_ptr=off(ws))[0] == -1
    assert b"16-byte aligned" in lib.nerrf_last_error()
    for H_ in (128, 512):
        assert _fwd(scorer, s, ln, tape, H_=H_)[0] == -1 and b"H == 256" in lib.nerrf_last_error()
        assert _bwd(scorer, s, ln, tape, dh, ws, H_=H_)[0] == -1 and b"H == 256" in lib.nerrf_last_error()
    # the refused calls wrote nothing: the tape still differentiates to the bits of a fresh round
    rc, got = _bwd(scorer, s, ln, tape, dh, ws)
    L.check(rc)
    _, fresh = _abi_round(scorer, s, ln, dh, *_buffers(B, T, D, 2))
    for k in got:
        assert torch.equal(got[k], fresh[k]), k


@gpu
def test_lengths_out_of_range_are_clamped_consistently():
    """Lengths above T give the bits of T and negative lengths the bits of 0, in hfin and in every gradient: the forward
    compares steps against the raw lengths, the backward clamps them, and the two must agree."""
    B, T, D = 45, 30, 16
    scorer = LSTMScorer(D, H, 2, seed=3).cuda()
    seq, lengths, _ = _batch(B, T, D, seed=3)
    wild = lengths.clone().to(torch.int32)
    wild[[4, 9, 17]] = torch.tensor([T + 1, 1000, 2 ** 31 - 1], dtype=torch.int32)
    wild[[5, 12, 30]] = torch.tensor([-1, -50, -2 ** 31], dtype=torch.int32)
    clamped = wild.clamp(0, T)
    s, dh = seq.cuda(), torch.randn(B, 2 * H, device="cuda")
    runs = [_abi_round(scorer, s, ln.cuda(), dh, *_buffers(B, T, D, 2)) for ln in (wild, clamped)]
    assert torch.equal(runs[0][0], runs[1][0]), "hfin"
    for k in runs[0][1]:
        assert torch.equal(runs[0][1][k], runs[1][1][k]), k
    assert not runs[0][0][[5, 12, 30]].any()
    assert not runs[0][1]["dseq"][[5, 12, 30]].any()


# --------------------------------------------------------------------------------------- reproducibility, tape reuse
def _library(scorer, seq, lengths, dlogit):
    scorer.zero_grad(set_to_none=True)
    x = seq.cuda().requires_grad_()
    (AG.lstm_logits(scorer, x, lengths.cuda()) * dlogit.cuda()).sum().backward()
    params = dict(scorer.named_parameters())
    out = {n: params[n].grad.detach().clone() for n in _names(scorer.num_layers)}
    out["dseq"] = x.grad.detach().clone()
    return out


def _same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), f"{what}: {k}"


@gpu
def test_tape_reuse_and_reproducibility(monkeypatch):
    """A scorer whose LSTMTape grew on a B = 4095 step gives a B = 37 step the bits of a fresh scorer, also with its
    tape and workspace filled with NaN first (stale contents are never read); two steps give the same bits; the
    training bits do not depend on NERRF_LSTM_ALGO (which selects the inference kernel only)."""
    small = _batch(37, 100, 16, seed=37)
    big = _batch(4095, 100, 16, seed=4095, lo=50)
    want = _library(LSTMScorer(seed=9).cuda(), *small)
    used = LSTMScorer(seed=9).cuda()
    _library(used, *big)
    tape = used._train_tape
    big_bytes = (tape._tape.numel(), tape._ws.numel())
    assert big_bytes == _sizes(4095, 100, 16, 2)
    _same(want, _library(used, *small), "after a B = 4095 step")
    assert (tape._tape.numel(), tape._ws.numel()) == big_bytes            # the buffers were reused, not reallocated
    tape._tape.fill_(0xFF)                                                 # every float NaN
    tape._ws.fill_(0xFF)
    _same(want, _library(used, *small), "NaN-filled tape and workspace")
    _same(want, _library(used, *small), "second step")
    for algo in ("umma", "ffma"):
        monkeypatch.setenv("NERRF_LSTM_ALGO", algo)
        _same(want, _library(used, *small), f"NERRF_LSTM_ALGO={algo}")


# ------------------------------------------------------------------------------------------- workspace sizes (CPU)
def test_train_workspace_is_a_function_of_the_shape_only(lib_built):
    """nerrf_lstm_train_workspace_bytes against bwd_plan and LstmTape restated: chunks of whole sequences, at most 32, and
    nothing that depends on the device."""
    lib = L.lib()
    tb, wb = C.c_size_t(), C.c_size_t()
    for B in (0, 1, 7, 8, 9, 31, 32, 33, 255, 256, 257, 1000, 4095, 4096, 4097, 100_000):
        for layers in (1, 2, 3):
            for D in (5, 16, 64, 1024):
                assert lib.nerrf_lstm_train_workspace_bytes(B, 100, D, H, layers, C.byref(tb), C.byref(wb)) == 0
                assert (tb.value, wb.value) == _sizes(B, 100, D, layers), (B, layers, D)
    assert _plan(512) == (16, 32) and _plan(1000) == (32, 32) and _plan(4095) == (128, 32) and _plan(257) == (9, 29)
    assert _plan(0) == (1, 1) and _plan(7) == (1, 7) and _plan(4097) == (129, 32)
