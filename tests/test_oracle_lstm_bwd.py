"""The hand-written BiLSTM backward oracle (oracle/lstm_bwd_ref.py) against torch.autograd in float64, over
torch.nn.LSTM + pack_padded_sequence and over the forward oracle oracle/lstm_ref.py: two independent witnesses of the
gradients the CUDA backward kernels (csrc/lstm_bwd.cu) are checked against.  Also: the new training entry points refuse
bad arguments before touching memory (CPU box: nothing is launched)."""
import ctypes
import math

import numpy as np
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence

from oracle import lstm_bwd_ref as B, lstm_ref as R

HID = 8          # the oracle is generic in H; the CUDA kernels are H = 256 only (tests/test_gpu_lstm_train.py)


def _case(D, T, L, seed, zero_len):
    rng = np.random.default_rng(seed)
    Bn = 6
    lengths = rng.integers(1, T + 1, Bn)
    lengths[0] = T; lengths[1] = 1
    if zero_len:
        lengths[2] = 0
    seq = rng.standard_normal((Bn, T, D))
    for b in range(Bn):
        seq[b, lengths[b]:] = 1e3                     # padded tail: never read
    dlogit = rng.standard_normal((Bn, 2))
    return R.make_params(D, HID, L, seed=seed), seq, lengths, dlogit


def _close(got, want):
    want = want.detach().numpy() if hasattr(want, "detach") else np.asarray(want)
    scale = max(1.0, float(np.abs(want).max()))
    assert np.allclose(got, want, rtol=1e-9, atol=1e-11 * scale), float(np.abs(got - want).max())


def _check(got, lstm_grads, head_W, head_b, seq):
    """lstm_grads[l][d] = (dW_ih, dW_hh, db_ih, db_hh) from autograd."""
    for l, dirs in enumerate(got["lstm"]):
        for d in range(2):
            for a, b in zip(dirs[d], lstm_grads[l][d]):
                _close(a, b)
    _close(got["head_W"], head_W); _close(got["head_b"], head_b); _close(got["seq"], seq)


@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("D", [5, 16])
@pytest.mark.parametrize("T", [1, 7, 30])
def test_oracle_equals_autograd_of_nn_lstm(L, D, T):
    P, seq, lengths, dlogit = _case(D, T, L, seed=10 * L + D + T, zero_len=False)
    m = R.to_nn_lstm(P, D, HID).double()
    head_W = P["head_W"].double().requires_grad_(); head_b = P["head_b"].double().requires_grad_()
    x = torch.from_numpy(seq).requires_grad_()
    packed = pack_padded_sequence(x, torch.from_numpy(lengths), batch_first=True, enforce_sorted=False)
    _, (hn, _) = m(packed)
    logit = torch.cat([hn[-2], hn[-1]], 1) @ head_W.t() + head_b
    (logit * torch.from_numpy(dlogit)).sum().backward()
    got = B.model_backward(P, seq, lengths, dlogit)
    _close(B.logits(P, seq, lengths), logit)
    grads = [[tuple(getattr(m, f"{n}_l{l}{sfx}").grad for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
              for sfx in ("", "_reverse")] for l in range(L)]
    _check(got, grads, head_W.grad, head_b.grad, x.grad)


def _ref_logits(params, seq, lengths):
    """oracle/lstm_ref.forward without the final sigmoid (autograd through the explicit cell loop)."""
    x = seq
    for fw, bw in params["lstm"]:
        of, hf = R.run_direction(x, lengths, *fw, reverse=False)
        ob, hb = R.run_direction(x, lengths, *bw, reverse=True)
        x = torch.cat([of, ob], 2)
    return torch.cat([hf, hb], 1) @ params["head_W"].t() + params["head_b"]


@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("D", [5, 16])
@pytest.mark.parametrize("T", [1, 7, 30])
def test_oracle_equals_autograd_of_the_forward_oracle(L, D, T):
    """Includes a zero-length sequence (pack_padded_sequence refuses those; the explicit loop does not)."""
    P, seq, lengths, dlogit = _case(D, T, L, seed=7 * L + D + 3 * T, zero_len=True)
    leaf = lambda t: t.double().requires_grad_()
    params = {"lstm": [[tuple(leaf(w) for w in d) for d in layer] for layer in P["lstm"]],
              "head_W": leaf(P["head_W"]), "head_b": leaf(P["head_b"])}
    x = torch.from_numpy(seq).requires_grad_()
    logit = _ref_logits(params, x, torch.from_numpy(lengths))
    (logit * torch.from_numpy(dlogit)).sum().backward()
    got = B.model_backward(P, seq, lengths, dlogit)
    _close(B.logits(P, seq, lengths), logit)
    grads = [[tuple(w.grad for w in d) for d in layer] for layer in params["lstm"]]
    _check(got, grads, params["head_W"].grad, params["head_b"].grad, x.grad)
    # the zero-length sequence contributes only through the head
    assert not np.any(got["seq"][2])


@pytest.mark.parametrize("batch", [1, 4, 8])
def test_sliced_oracle_equals_the_whole_batch(batch):
    """logits / model_backward with batch= (the form the scale tests use) against one pass over the whole batch: logits
    and dseq concatenate, parameter gradients sum.  The slice boundaries at 4 and 8 fall between a full-length and a
    zero-length sequence."""
    T, D, L = 9, 5, 2
    P = R.make_params(D, HID, L, seed=17)
    rng = np.random.default_rng(18)
    lengths = np.array([3, 1, 6, T, 0, 2, 5, 0, T, 4, 0])
    seq = rng.standard_normal((lengths.size, T, D))
    dlogit = rng.standard_normal((lengths.size, 2))
    whole = B.model_backward(P, seq, lengths, dlogit)
    part = B.model_backward(P, seq, lengths, dlogit, batch=batch)

    def near(a, b):
        assert a.shape == b.shape
        assert np.abs(a - b).max() <= 1e-12 * max(1.0, float(np.abs(b).max()))
    want_logits = B.logits(P, seq, lengths)
    near(B.logits(P, seq, lengths, batch=batch), want_logits)
    near(part["logits"], want_logits); near(whole["logits"], want_logits)
    near(part["seq"], whole["seq"]); near(part["head_W"], whole["head_W"]); near(part["head_b"], whole["head_b"])
    for la, lb in zip(part["lstm"], whole["lstm"]):
        for da, db in zip(la, lb):
            for a, b in zip(da, db):
                near(a, b)
    assert not part["seq"][4].any() and not part["seq"][7].any()


def test_hand_computed_h1_t2():
    """H = 1, D_in = 1, T = 2, one layer: the forward direction's gradients written out as scalars, and checked against
    central differences of the scalar forward."""
    sig = lambda v: 1.0 / (1.0 + math.exp(-v))
    wih = [0.3, -0.2, 0.5, 0.1]; whh = [0.4, 0.2, -0.3, 0.6]; bias = [0.05, -0.1, 0.2, 0.0]     # gates i, f, g, o
    x0, x1 = 0.7, -1.2
    hw = [0.9, -0.4]                                  # head row 0 over [h_fwd || h_bwd]
    bw = ([0.1, 0.2, 0.3, 0.4], [0.5, -0.5, 0.25, -0.25], [0.0, 0.1, 0.0, 0.1], [0.0] * 4)

    def fwd_dir(wih_, whh_, b_):
        h, c, saved = 0.0, 0.0, []
        for x in (x0, x1):
            a = [wih_[k] * x + whh_[k] * h + b_[k] for k in range(4)]
            i, f, g, o = sig(a[0]), sig(a[1]), math.tanh(a[2]), sig(a[3])
            c_prev, h_prev = c, h
            c = f * c + i * g
            h = o * math.tanh(c)
            saved.append((i, f, g, o, c, c_prev, h_prev))
        return h, saved

    _, saved = fwd_dir(wih, whh, bias)
    e = hw[0]                                         # d logit0 / d h_fwd_final
    (i0, f0, g0, o0, c0, _, _), (i1, f1, g1, o1, c1, cp1, h0) = saved
    dc1 = e * o1 * (1 - math.tanh(c1) ** 2)
    da1 = [dc1 * g1 * i1 * (1 - i1), dc1 * cp1 * f1 * (1 - f1), dc1 * i1 * (1 - g1 * g1), e * math.tanh(c1) * o1 * (1 - o1)]
    dh0 = sum(da1[k] * whh[k] for k in range(4))
    dc0 = dc1 * f1 + dh0 * o0 * (1 - math.tanh(c0) ** 2)
    da0 = [dc0 * g0 * i0 * (1 - i0), 0.0, dc0 * i0 * (1 - g0 * g0), dh0 * math.tanh(c0) * o0 * (1 - o0)]
    want_wih = [da0[k] * x0 + da1[k] * x1 for k in range(4)]
    want_whh = [da1[k] * h0 for k in range(4)]
    want_b = [da0[k] + da1[k] for k in range(4)]

    col = lambda v: np.array(v)[:, None]
    P = {"lstm": [[(col(wih), col(whh), np.array(bias), np.zeros(4)), (col(bw[0]), col(bw[1]), np.array(bw[2]), np.array(bw[3]))]],
         "head_W": np.array([hw, [0.0, 0.0]]), "head_b": np.zeros(2)}
    seq = np.array([[[x0], [x1]]]); lengths = np.array([2])
    got = B.model_backward(P, seq, lengths, np.array([[1.0, 0.0]]))
    dW_ih, dW_hh, db_ih, db_hh = got["lstm"][0][0]
    assert np.allclose(dW_ih[:, 0], want_wih, rtol=1e-12, atol=1e-15)
    assert np.allclose(dW_hh[:, 0], want_whh, rtol=1e-12, atol=1e-15)
    assert np.allclose(db_ih, want_b, rtol=1e-12, atol=1e-15) and np.array_equal(db_ih, db_hh)
    # central differences of the scalar forward
    eps = 1e-6
    for k in range(4):
        for vec, want in ((wih, want_wih), (whh, want_whh), (bias, want_b)):
            up = list(vec); dn = list(vec); up[k] += eps; dn[k] -= eps
            args = lambda v: (v if vec is wih else wih, v if vec is whh else whh, v if vec is bias else bias)
            num = (fwd_dir(*args(up))[0] - fwd_dir(*args(dn))[0]) / (2 * eps) * e
            assert abs(num - want[k]) < 1e-8


# ---------------------------------------------------------------- argument errors of the C-ABI training entry points
def _fake(n):
    return ctypes.c_void_p(n << 20)


def _ptrs(n, base):
    arr = (ctypes.c_void_p * n)()
    for i in range(n):
        arr[i] = (base + i) << 20
    return arr


def test_training_entry_points_refuse_bad_arguments(lib_built):
    from nerrf_b200 import _lib
    h = _lib.lib()
    tb, wb = ctypes.c_size_t(), ctypes.c_size_t()
    assert h.nerrf_lstm_train_workspace_bytes(4, 100, 16, 128, 2, ctypes.byref(tb), ctypes.byref(wb)) == -1   # H != 256
    assert b"H == 256" in h.nerrf_last_error()
    assert h.nerrf_lstm_train_workspace_bytes(4, 100, 16, 256, 2, None, ctypes.byref(wb)) == -1
    assert h.nerrf_lstm_train_workspace_bytes(4, 100, 16, 256, 2, ctypes.byref(tb), ctypes.byref(wb)) == 0
    # 2 layers x (out 2H + gates 2*4H + cells 2H) floats per row
    assert tb.value == 2 * 4 * 100 * 12 * 256 * 4 and wb.value > 4 * 100 * 2 * 256 * 4
    need_tape, need_ws = tb.value, wb.value

    W = lambda: _ptrs(4, 40)
    # forward_train(seq, len, B, T, D_in, H, L, Wih_t, Whh_t, bias, hfin_out, tape, tape_bytes, stream)
    fwd = lambda H=256, seq=_fake(1), tape=_fake(9), tape_bytes=need_tape, hfin=_fake(8): h.nerrf_lstm_forward_train(
        seq, _fake(2), 4, 100, 16, H, 2, W(), W(), W(), hfin, tape, tape_bytes, None)
    assert fwd(H=255) == -1
    assert fwd(seq=None) == -1 and b"null" in h.nerrf_last_error()
    assert fwd(hfin=None) == -1
    assert fwd(tape=ctypes.c_void_p((9 << 20) + 4)) == -1 and b"aligned" in h.nerrf_last_error()
    assert fwd(tape_bytes=need_tape - 1) == -4 and b"tape too small" in h.nerrf_last_error()
    assert h.nerrf_lstm_forward_train(_fake(1), _fake(2), 4, 100, 16, 256, 2, None, W(), W(), _fake(8), _fake(9), need_tape,
                                      None) == -1

    # backward(seq, len, B, T, D_in, H, L, W_ih, W_hh, tape, tape_bytes, dhfin, dseq, dW_ih, dW_hh, db, ws, ws_bytes, stream)
    def bwd(H=256, dhfin=_fake(10), tape_bytes=need_tape, ws_bytes=need_ws, dW=True):
        return h.nerrf_lstm_backward(_fake(1), _fake(2), 4, 100, 16, H, 2, W(), W(), _fake(9), tape_bytes, dhfin, None,
                                     W() if dW else None, W(), W(), _fake(11), ws_bytes, None)
    assert bwd(H=512) == -1 and b"H == 256" in h.nerrf_last_error()
    assert bwd(dhfin=None) == -1
    assert bwd(dW=False) == -1
    assert bwd(tape_bytes=need_tape // 2) == -4 and b"tape too small" in h.nerrf_last_error()
    assert bwd(ws_bytes=need_ws - 1) == -4 and b"workspace too small" in h.nerrf_last_error()
