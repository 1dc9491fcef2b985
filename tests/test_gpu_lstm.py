"""lstm.forward CUDA path vs the oracle (needs an H100).  The wgmma path (csrc/lstm_umma.cu) is the default; the fp32
CUDA-core kernel (csrc/lstm.cu, NERRF_LSTM_ALGO=ffma) stays as an independent cross-check of it."""
import pytest
import torch

from nerrf_b200.ai.models import lstm
from oracle import lstm_ref as LR
from gpu_util import assert_close_fp32

pytestmark = pytest.mark.gpu

# VERDICT r1 next #3: B in {1, 5, 127, 128, 129, 700, 4096} x T in {1, 7, 100} (the 64-sequence tile boundary at 63/64/65
# too); every batch carries a zero-length sequence, a full-length one and ragged ones.  B=4096 / T=100 is checked on a
# sample of rows (the explicit-loop oracle would need minutes for all of them).
MATRIX = [(1, 1), (1, 100), (5, 7), (63, 7), (64, 7), (65, 7), (127, 1), (127, 100), (128, 7), (129, 100), (700, 7), (700, 100)]


def _batch(B, T, seed, D=16):
    g = torch.Generator().manual_seed(seed)
    seq = torch.randn(B, T, D, generator=g)
    lengths = torch.randint(0, T + 1, (B,), generator=g)
    lengths[0] = T
    if B > 1:
        lengths[1] = 0                                   # an empty sequence: its state never leaves zero
    if B > 2:
        lengths[2] = 1
    return seq, lengths


@pytest.mark.parametrize("algo", ["umma", "ffma"])
@pytest.mark.parametrize("B,T", MATRIX)
def test_lstm_parity(B, T, algo, monkeypatch):
    monkeypatch.setenv("NERRF_LSTM_ALGO", algo)
    model = lstm.LSTMScorer(16, 256, 2, seed=3).cuda()
    seq, lengths = _batch(B, T, B * 1000 + T)
    got = model(seq.cuda(), lengths.cuda())
    want = LR.forward(model.oracle_params(), seq, lengths)
    assert got.shape == (B, 2)
    assert float((got.cpu() - want).abs().max()) < 1e-5, f"lstm {algo} B={B} T={T}"      # fp32-equivalent (measured ~1e-7)
    assert_close_fp32(got, want, rtol=1e-4, atol_rms=1e-5, what=f"lstm {algo} B={B} T={T}")
    if B > 1:                                           # zero-length sequence -> head of the zero state
        z = LR.forward(model.oracle_params(), seq[1:2], torch.zeros(1, dtype=torch.int64))
        assert float((got[1].cpu() - z[0]).abs().max()) < 1e-6


@pytest.mark.parametrize("layers,D", [(1, 16), (3, 16), (2, 5), (2, 32), (2, 64)])
def test_lstm_layer_counts_and_input_widths(layers, D, monkeypatch):
    monkeypatch.setenv("NERRF_LSTM_ALGO", "umma")
    model = lstm.LSTMScorer(D, 256, layers, seed=5).cuda()
    seq, lengths = _batch(70, 9, 77, D=D)
    got = model(seq.cuda(), lengths.cuda())
    want = LR.forward(model.oracle_params(), seq, lengths)
    assert float((got.cpu() - want).abs().max()) < 1e-5


def test_full_size_batch_sampled_against_oracle_and_cross_checked():
    """B=4096 / T=100 (the bench shape): rows are independent, so a 96-row sample through the oracle checks them; the
    whole batch is cross-checked against the fp32 CUDA-core kernel."""
    import os
    model = lstm.LSTMScorer().cuda()
    seq, lengths = _batch(4096, 100, 4096100)
    os.environ["NERRF_LSTM_ALGO"] = "umma"
    try:
        got = model(seq.cuda(), lengths.cuda()).cpu()
        os.environ["NERRF_LSTM_ALGO"] = "ffma"
        ref = model(seq.cuda(), lengths.cuda()).cpu()
    finally:
        os.environ.pop("NERRF_LSTM_ALGO", None)
    assert float((got - ref).abs().max()) < 2e-6
    rows = torch.cat([torch.arange(0, 40), torch.arange(2040, 2072), torch.arange(4072, 4096)])
    want = LR.forward(model.oracle_params(), seq[rows], lengths[rows])
    assert float((got[rows] - want).abs().max()) < 1e-5
    assert torch.equal(got, model(seq.cuda(), lengths.cuda()).cpu())             # deterministic


def test_padding_is_ignored_and_module_level_forward():
    model = lstm.LSTMScorer().cuda()
    seq = torch.randn(9, 100, 16, device="cuda")
    lengths = torch.tensor([100, 3, 50, 1, 99, 100, 17, 2, 64], device="cuda")
    a = model(seq, lengths)
    seq2 = seq.clone()
    for b in range(9):
        seq2[b, int(lengths[b]):] = 1e6          # garbage in the padded tail
    assert torch.equal(a, model(seq2, lengths))
    assert torch.equal(a, lstm.forward(seq, lengths, model))
    assert (a > 0).all() and (a < 1).all()
