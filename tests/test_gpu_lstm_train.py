"""BiLSTM training through the library's kernels (needs an H100): the saved-activation forward
(`nerrf_lstm_forward_train`) and the backward-through-time (`nerrf_lstm_backward`, csrc/lstm_bwd.cu) behind
nerrf_b200.ai.autograd.LSTMFn, against the hand-written fp64 oracle (oracle/lstm_bwd_ref.py, itself pinned to autograd in
tests/test_oracle_lstm_bwd.py)."""
import numpy as np
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence

from nerrf_b200.ai import autograd as AG
from nerrf_b200.ai import train as T
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.ai.models.lstm import LSTMScorer
from oracle import lstm_bwd_ref as LB

pytestmark = pytest.mark.gpu

RTOL, ATOL_RMS = 2e-4, 2e-5        # the _grad_close bound of tests/test_gpu_train.py


def _batch(B, Tn, D, seed, garbage=0.0):
    g = torch.Generator().manual_seed(seed)
    seq = torch.randn(B, Tn, D, generator=g)
    lengths = torch.randint(0, Tn + 1, (B,), generator=g)
    lengths[0] = Tn
    if B > 1:
        lengths[1] = 0
    if B > 2:
        lengths[2] = 1
    for b in range(B):
        seq[b, int(lengths[b]):] = garbage
    dlogit = torch.randn(B, 2, generator=g)
    return seq, lengths, dlogit


def _names(L):
    return [f"lstm.{n}_l{l}{sfx}" for l in range(L) for sfx in ("", "_reverse")
            for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")] + ["head.weight", "head.bias"]


def _oracle(scorer, seq, lengths, dlogit):
    w = LB.model_backward(scorer.oracle_params(), seq, lengths, dlogit)
    flat = [g for layer in w["lstm"] for d in layer for g in d] + [w["head_W"], w["head_b"]]
    return dict(zip(_names(scorer.num_layers), flat)), w["seq"]


def _library(scorer, seq, lengths, dlogit):
    scorer.zero_grad(set_to_none=True)
    x = seq.cuda().requires_grad_()
    (AG.lstm_logits(scorer, x, lengths.cuda()) * dlogit.cuda()).sum().backward()
    params = dict(scorer.named_parameters())
    return {n: params[n].grad.detach().clone() for n in _names(scorer.num_layers)}, x.grad.detach().clone()


def _torch_fp32(scorer, seq, lengths, dlogit):
    """fp32 CPU torch.nn.LSTM autograd of the same case: what the library is allowed to be as far from the oracle as.
    pack_padded_sequence refuses zero-length sequences: they are left out, and their exact contribution (dlogit to the head
    bias, nothing else) is added back."""
    cpu = LSTMScorer(scorer.in_dim, 256, scorer.num_layers, seed=None)
    cpu.load_state_dict({k: v.detach().cpu() for k, v in scorer.state_dict().items()})
    keep = lengths > 0
    x = seq[keep].clone().requires_grad_()
    packed = pack_padded_sequence(x, lengths[keep], batch_first=True, enforce_sorted=False)
    _, (hn, _) = cpu.lstm(packed)
    (cpu.head(torch.cat([hn[-2], hn[-1]], 1)) * dlogit[keep]).sum().backward()
    params = dict(cpu.named_parameters())
    grads = {n: params[n].grad.clone() for n in _names(cpu.num_layers)}
    grads["head.bias"] += dlogit[~keep].sum(0)
    dseq = torch.zeros_like(seq)
    dseq[keep] = x.grad
    return grads, dseq


def _ratio(got, want):
    """max |got - want| / (RTOL |want| + ATOL_RMS rms(want)): <= 1 is inside the _grad_close bound."""
    got = np.asarray(got.detach().double().cpu().numpy() if hasattr(got, "detach") else got, np.float64)
    want = np.asarray(want, np.float64)
    rms = float(np.sqrt((want ** 2).mean())) if want.size else 0.0
    return float((np.abs(got - want) / (RTOL * np.abs(want) + ATOL_RMS * max(rms, 1e-30))).max())


CASES = [(1, 1, 2, 16), (1, 100, 2, 16), (7, 7, 2, 16), (8, 7, 2, 16), (9, 100, 2, 16), (33, 7, 2, 16), (100, 100, 2, 16),
         (256, 100, 2, 16), (9, 100, 1, 16), (9, 100, 3, 16), (33, 30, 2, 5), (33, 30, 2, 32), (20, 50, 3, 5)]


@pytest.mark.parametrize("B,Tn,L,D", CASES)
def test_gradients_match_the_fp64_oracle(B, Tn, L, D):
    """Every LSTMScorer parameter and dseq, random dlogit on both head outputs; lengths 0, 1 and T in every batch of 3 or
    more.  Bound: the _grad_close form, widened only as far as fp32 torch.nn.LSTM autograd itself lands on the same case."""
    scorer = LSTMScorer(D, 256, L, seed=B + Tn + L).cuda()
    seq, lengths, dlogit = _batch(B, Tn, D, seed=1000 * B + Tn + L)
    want, want_seq = _oracle(scorer, seq, lengths, dlogit)
    got, got_seq = _library(scorer, seq, lengths, dlogit)
    ref, ref_seq = _torch_fp32(scorer, seq, lengths, dlogit)
    report = []
    for n in want:
        allowed = max(1.0, _ratio(ref[n], want[n]))
        r = _ratio(got[n], want[n])
        report.append(f"{n} {r:.3f} (torch {allowed:.3f})")
        assert r <= allowed, f"{n}: error ratio {r:.3f} > {allowed:.3f} (B={B} T={Tn} L={L} D={D})"
    allowed = max(1.0, _ratio(ref_seq, want_seq))
    r = _ratio(got_seq, want_seq)
    report.append(f"dseq {r:.3f} (torch {allowed:.3f})")
    assert r <= allowed, f"dseq: error ratio {r:.3f} > {allowed:.3f}"
    print(f"B={B} T={Tn} L={L} D={D}: " + ", ".join(report))


@pytest.mark.parametrize("algo,tol", [("ffma", 1e-6), ("umma", 2e-6)])
def test_forward_train_matches_inference(algo, tol, monkeypatch):
    """The head applied to forward_train's hfin gives what LSTMScorer.forward (the inference kernels) gives."""
    monkeypatch.setenv("NERRF_LSTM_ALGO", algo)
    scorer = LSTMScorer().cuda()
    seq, lengths, _ = _batch(300, 100, 16, seed=5)
    with torch.no_grad():
        probs = scorer(seq.cuda(), lengths.cuda())
        train_probs = torch.sigmoid(AG.lstm_logits(scorer, seq.cuda(), lengths.cuda()))
    assert float((train_probs - probs).abs().max()) <= tol


def test_padding_is_ignored_and_backward_is_deterministic():
    scorer = LSTMScorer().cuda()
    seq, lengths, dlogit = _batch(37, 60, 16, seed=9)
    g0, s0 = _library(scorer, seq, lengths, dlogit)
    junk = seq.clone()
    for b in range(37):
        junk[b, int(lengths[b]):] = 1e6                  # garbage in the padded tail (all of the zero-length sequence)
    g1, s1 = _library(scorer, junk, lengths, dlogit)
    for n in g0:
        assert torch.equal(g0[n], g1[n]), n
    assert torch.equal(s0, s1)
    for b in range(37):
        assert not s1[b, int(lengths[b]):].any()         # dseq exactly 0 at padded steps
    # the zero-length sequence (row 1) contributes only through the head: no input gradient, zero final state
    assert not s1[1].any()
    with torch.no_grad():
        hfin = AG.LSTMFn.apply(seq.cuda(), lengths.cuda(), AG.LSTMTape(), 2, False, *AG.lstm_params(scorer))
    assert not hfin[1].any()
    # a second backward gives identical bits
    g2, s2 = _library(scorer, seq, lengths, dlogit)
    for n in g0:
        assert torch.equal(g0[n], g2[n]), n
    assert torch.equal(s0, s2)


def test_two_forwards_before_backward_keep_their_tapes():
    """A second forward while the first one's backward is pending gets a tape of its own."""
    scorer = LSTMScorer().cuda()
    seq, lengths, dlogit = _batch(17, 30, 16, seed=4)
    want, _ = _library(scorer, seq, lengths, dlogit)
    scorer.zero_grad(set_to_none=True)
    a = (AG.lstm_logits(scorer, seq.cuda(), lengths.cuda()) * dlogit.cuda()).sum()
    seq2, lengths2, dlogit2 = _batch(17, 30, 16, seed=5)
    b = (AG.lstm_logits(scorer, seq2.cuda(), lengths2.cuda()) * dlogit2.cuda()).sum()
    a.backward()
    params = dict(scorer.named_parameters())
    for n in want:
        assert torch.equal(params[n].grad, want[n]), n
    b.backward()
    with pytest.raises(RuntimeError):
        a.backward()                                     # the graph was freed (and the tape consumed)


def test_training_through_the_library_lstm_passes_the_gate():
    """ai.train with device='cuda', lstm_backward='library': both models through the library's kernels; ROC-AUC >= 0.90
    on a held-out toy trace, the LSTM scored through the inference kernels (LSTMScorer.forward)."""
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3, device="cuda", lstm_backward="library")
    ex = T._to(T.make_example(901, n_files=30, benign_files=40), "cuda")
    _, score = model(ex["x"], ex["rowptr"], ex["col"], ex["ew"])
    probs = scorer(ex["seq"], ex["lengths"])
    files = ex["is_file"].cpu().numpy()
    gnn = T.roc_auc(score.cpu().numpy()[files], ex["label"].cpu().numpy()[files])
    lstm_auc = T.roc_auc(probs[:, 0].cpu().numpy(), ex["seq_label"].cpu().numpy())
    print(f"held-out ROC-AUC: GNN {gnn:.4f}, LSTM {lstm_auc:.4f}")
    assert gnn >= 0.90 and lstm_auc >= 0.90


def test_default_training_path_never_reaches_the_library_lstm(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("the default lstm_backward='torch' must not call autograd.lstm_logits")
    monkeypatch.setattr(AG, "lstm_logits", refuse)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 101), windows=0), epochs=1, device="cuda")
    with pytest.raises(ValueError):
        T.train(model, scorer, [], epochs=1, device="cuda", lstm_backward="cudnn")
