"""Statements of the BiLSTM sequence-step attributions (DESIGN.md 1.2.1) for the tests: the float64 oracle, built on
oracle/lstm_bwd_ref.py, and the float32 restatement of what nerrf_lstm_explain_steps computes from a given dseq."""
import numpy as np

from oracle import lstm_bwd_ref as LB


def sequence_attributions(params, seq, lengths, batch=None):
    """float64: -> (z [B] encrypt logits, a [B, T, D] with a[b,t,d] = x[b,t,d] * dz_b/dx[b,t,d], 0 at t >= len[b])"""
    x = np.asarray(seq.cpu().numpy() if hasattr(seq, "cpu") else seq, np.float64)
    ln = np.asarray(lengths.cpu().numpy() if hasattr(lengths, "cpu") else lengths, np.int64)
    dlogit = np.zeros((x.shape[0], 2))
    dlogit[:, 0] = 1.0
    g = LB.model_backward(params, x, ln, dlogit, batch=batch)
    valid = np.arange(x.shape[1])[None, :] < ln[:, None]
    return g["logits"][:, 0], np.where(valid[..., None], x * g["seq"], 0.0)


def step_attr_f32(seq, dseq):
    """float32: a_t = sum_d seq * dseq, each product rounded, summed left to right (d ascending) -> [..., T]"""
    p = np.asarray(seq, np.float32) * np.asarray(dseq, np.float32)
    s = p[..., 0].copy()
    for d in range(1, p.shape[-1]):
        s = s + p[..., d]
    return s


def dominant_feature(seq, dseq):
    """argmax_d |seq * dseq| (float32 products), ties to the lower d; -1 when every term is 0 (NaN terms never win)"""
    m = np.abs(np.asarray(seq, np.float32) * np.asarray(dseq, np.float32))
    m = np.where(np.isnan(m), 0.0, m)
    return np.where(m.max(-1) > 0, m.argmax(-1), -1)


def top_steps(a_t, length, k):
    """the k steps t < length of largest |a_t|, ties to the lower t, NaN below every number"""
    key = np.abs(np.asarray(a_t, np.float64)[:length])
    key = np.where(np.isnan(key), -0.5, key)
    return np.lexsort((np.arange(length), -key))[:k]
