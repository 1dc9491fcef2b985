"""BiLSTM BACKWARD-THROUGH-TIME oracle (numpy, float64 by default; test infra -- see oracle/__init__.py).

Reference surface: the BiLSTM half of ``ai/train.py`` "joint GNN+LSTM training script" (README.md:75 -- named, never
written).  The forward spec is oracle/lstm_ref.py (frozen, SURVEY.md 8a row a4): torch gate order (i, f, g, o), valid
steps t < len[b] (packed-sequence semantics: a padded step leaves h and c unchanged and outputs 0), a bidirectional
stack, head = Linear(2H, 2) on [h_fwd_final || h_bwd_final] of the top layer.

The backward written out by hand, per layer, per direction, per step in reverse direction order (the chain rule of
``h = where(valid, h', h);  c = where(valid, c', c);  out_t = where(valid, h', 0)``):

    valid:   dh' = dh + dout_t;   dc' = dc + dh' o (1 - tanh^2 c')
             da  = [dc' g i(1-i),  dc' c_{t-1} f(1-f),  dc' i (1-g^2),  dh' tanh(c') o(1-o)]      (pre-activations)
             dW_ih += da^T x_t;   dW_hh += da^T h_{t-1};   db += da;   dx_t += da W_ih
             dh <- da W_hh;   dc <- dc' f
    padded:  dh, dc pass through unchanged

The final state gradient (from the head) enters as the initial dh.  tests/test_oracle_lstm_bwd.py pins every function
here against torch.autograd over torch.nn.LSTM + pack_padded_sequence and over oracle/lstm_ref.py, both in float64 (two
independent witnesses: this file never builds an autograd graph).
"""
import numpy as np


def _sig(x):
    with np.errstate(over="ignore"):            # exp overflow -> 0, the correct limit
        return 1.0 / (1.0 + np.exp(-x))


def _arr(t, dtype):
    return np.asarray(t.detach().cpu().numpy() if hasattr(t, "detach") else t, dtype)


def direction_forward(x, lengths, W_ih, W_hh, b_ih, b_hh, reverse):
    """x [B,T,D] -> (out [B,T,H], h_final [B,H], tape) with the per-step gates / cells the backward needs."""
    B, T, _ = x.shape
    H = W_hh.shape[1]
    h = np.zeros((B, H), x.dtype); c = np.zeros((B, H), x.dtype)
    out = np.zeros((B, T, H), x.dtype)
    tape = {k: np.zeros((B, T, n * H), x.dtype) for k, n in (("gates", 4), ("c", 1), ("h_prev", 1), ("c_prev", 1))}
    for t in (range(T - 1, -1, -1) if reverse else range(T)):
        valid = (lengths > t)[:, None]
        a = x[:, t] @ W_ih.T + b_ih + h @ W_hh.T + b_hh
        i, f, g, o = _sig(a[:, :H]), _sig(a[:, H:2 * H]), np.tanh(a[:, 2 * H:3 * H]), _sig(a[:, 3 * H:])
        c2 = f * c + i * g
        h2 = o * np.tanh(c2)
        tape["gates"][:, t] = np.concatenate([i, f, g, o], 1)
        tape["c"][:, t] = c2; tape["h_prev"][:, t] = h; tape["c_prev"][:, t] = c
        h = np.where(valid, h2, h); c = np.where(valid, c2, c)
        out[:, t] = np.where(valid, h2, 0.0)
    return out, h, tape


def direction_backward(x, lengths, W_ih, W_hh, tape, dout, dh_final, reverse):
    """Gradients of sum(dout * out) + sum(dh_final * h_final) of one direction -> (dx, dW_ih, dW_hh, db)."""
    B, T, _ = x.shape
    H = W_hh.shape[1]
    dh = np.array(dh_final, x.dtype, copy=True); dc = np.zeros((B, H), x.dtype)
    dx = np.zeros_like(x); dW_ih = np.zeros_like(W_ih); dW_hh = np.zeros_like(W_hh); db = np.zeros(4 * H, x.dtype)
    for t in (range(T) if reverse else range(T - 1, -1, -1)):
        valid = (lengths > t)[:, None]
        gt = tape["gates"][:, t]
        i, f, g, o = gt[:, :H], gt[:, H:2 * H], gt[:, 2 * H:3 * H], gt[:, 3 * H:]
        tc = np.tanh(tape["c"][:, t])
        dh2 = np.where(valid, dh + dout[:, t], 0.0)
        dc2 = np.where(valid, dc, 0.0) + dh2 * o * (1.0 - tc * tc)
        da = np.concatenate([dc2 * g * i * (1 - i), dc2 * tape["c_prev"][:, t] * f * (1 - f), dc2 * i * (1 - g * g),
                             dh2 * tc * o * (1 - o)], 1)
        dW_ih += da.T @ np.where(valid, x[:, t], 0.0)
        dW_hh += da.T @ tape["h_prev"][:, t]
        db += da.sum(0)
        dx[:, t] += da @ W_ih
        dh = np.where(valid, da @ W_hh, dh)
        dc = np.where(valid, dc2 * f, dc)
    return dx, dW_ih, dW_hh, db


def _layers(params, dtype):
    return [[tuple(_arr(w, dtype) for w in d) for d in layer] for layer in params["lstm"]]


def _slices(n, batch):
    """Consecutive slices of at most `batch` sequences covering [0, n), or None when one pass does (batch None or >= n).
    Sequences are independent, so logits and dseq of a batch are those of its slices side by side, and the parameter
    gradients are the sum of the slices' gradients: slicing bounds the float64 tape (~5.7 MB per 100-step sequence of a
    2-layer H = 256 stack) without changing what is computed."""
    if batch is None or batch >= n:
        return None
    if batch < 1:
        raise ValueError("batch must be >= 1")
    return [slice(s, min(s + batch, n)) for s in range(0, n, batch)]


def logits(params, seq, lengths, dtype=np.float64, batch=None):
    """Head logits [B,2] (pre-sigmoid) = [h_fwd_final || h_bwd_final] head_W^T + head_b.  batch: evaluate `batch`
    sequences at a time (same result; bounds memory)."""
    x = _arr(seq, dtype); lengths = np.asarray(_arr(lengths, np.int64))
    parts = _slices(x.shape[0], batch)
    if parts is not None:
        return np.concatenate([logits(params, x[s], lengths[s], dtype) for s in parts], 0)
    hf = hb = None
    for fw, bw in _layers(params, dtype):
        of, hf, _ = direction_forward(x, lengths, *fw, reverse=False)
        ob, hb, _ = direction_forward(x, lengths, *bw, reverse=True)
        x = np.concatenate([of, ob], 2)
    return np.concatenate([hf, hb], 1) @ _arr(params["head_W"], dtype).T + _arr(params["head_b"], dtype)


def model_backward(params, seq, lengths, dlogit, dtype=np.float64, batch=None):
    """Gradients of sum(dlogit * logits(params, seq, lengths)) w.r.t. every parameter and seq.  params as
    oracle/lstm_ref.py (numpy arrays or torch tensors).  -> dict(lstm=[[(dW_ih, dW_hh, db_ih, db_hh) fwd, (...) bwd]
    per layer], head_W, head_b, seq, logits); db_ih == db_hh (the two biases enter the gates as one sum); logits are
    those of logits(), from the same forward pass.  batch: differentiate `batch` sequences at a time and sum the parameter
    gradients over the slices in slice order (bounds memory)."""
    x = _arr(seq, dtype); lengths = np.asarray(_arr(lengths, np.int64))
    parts = _slices(x.shape[0], batch)
    if parts is not None:
        dlogit = _arr(dlogit, dtype)
        out = None
        for s in parts:
            g = model_backward(params, x[s], lengths[s], dlogit[s], dtype)
            if out is None:
                out = g
                out["seq"], out["logits"] = [g["seq"]], [g["logits"]]
                continue
            out["head_W"] += g["head_W"]; out["head_b"] += g["head_b"]
            out["seq"].append(g["seq"]); out["logits"].append(g["logits"])
            out["lstm"] = [[tuple(a + b for a, b in zip(da, db)) for da, db in zip(la, lb)]
                           for la, lb in zip(out["lstm"], g["lstm"])]
        out["seq"], out["logits"] = np.concatenate(out["seq"], 0), np.concatenate(out["logits"], 0)
        return out
    layers = _layers(params, dtype)
    B, T, _ = x.shape
    H = layers[0][0][1].shape[1]
    ins, tapes = [], []
    for fw, bw in layers:
        of, hf, tf = direction_forward(x, lengths, *fw, reverse=False)
        ob, hb, tb = direction_forward(x, lengths, *bw, reverse=True)
        ins.append(x); tapes.append((tf, tb))
        x = np.concatenate([of, ob], 2)
    feat = np.concatenate([hf, hb], 1)
    dlogit = _arr(dlogit, dtype)
    head_W = _arr(params["head_W"], dtype)
    out = {"head_W": dlogit.T @ feat, "head_b": dlogit.sum(0), "lstm": [None] * len(layers),
           "logits": feat @ head_W.T + _arr(params["head_b"], dtype)}
    dfeat = dlogit @ head_W
    dout = np.zeros((B, T, 2 * H), dtype)
    for l in reversed(range(len(layers))):
        top = l == len(layers) - 1
        grads, din = [], 0.0
        for d, reverse in ((0, False), (1, True)):
            W_ih, W_hh = layers[l][d][0], layers[l][d][1]
            dh_final = dfeat[:, d * H:(d + 1) * H] if top else np.zeros((B, H), dtype)
            dx, dW_ih, dW_hh, db = direction_backward(ins[l], lengths, W_ih, W_hh, tapes[l][d], dout[:, :, d * H:(d + 1) * H],
                                                      dh_final, reverse)
            grads.append((dW_ih, dW_hh, db, db.copy()))
            din = din + dx
        out["lstm"][l] = grads
        dout = din
    out["seq"] = dout
    return out
