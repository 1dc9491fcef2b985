"""Exact statement of the window-graph model inputs: per-node features, per-file LSTM sequences and per-pair edge labels,
over plain event columns (node ids, slots, byte counts, times, path flags) in time order.

It is the statement the device kernels of csrc/graph.cu are checked against (tests/test_gpu_window_kernels.py) and is
itself checked against the event-by-event spec graph.graph_from_events / pipeline.file_sequences
(tests/test_window_statement_cpu.py).  It shares no code with the vectorised host twins (ingest.graph_from_columns,
ingest.sequences_core): integer quantities stay integers, every float column is computed in float64 from them in the
order the kernels use and rounded to float32 once.

A byte count is the wire's uint64 clamped to graph.MAX_RW_COUNT; a node's byte sum is an exact integer.
"""
from __future__ import annotations

import numpy as np

MAX_RW_COUNT = 0x7ffff000          # Linux's per-call read / write cap (graph.MAX_RW_COUNT, restated here on purpose)
PATH_LOCKBIT, PATH_NOTE, PATH_TMP = 1, 2, 4
D_IN = 16


def clamped(nbytes) -> np.ndarray:
    """uint64 byte counts (any integer dtype holding the wire's bits) -> int64, clamped to MAX_RW_COUNT"""
    b = np.asarray(nbytes)
    if b.dtype != np.uint64:
        b = b.astype(np.int64).view(np.uint64)
    return np.minimum(b, np.uint64(MAX_RW_COUNT)).astype(np.int64)


def node_accumulate(node_p, node_f, node_g, t, slot, nbytes, pflags, n_nodes):
    """The integer per-node state: cnt int64 [N, 8], deg int64 [N], bytes (Python ints) [N], first / last float64 [N],
    flags int64 [N] (NERRF_PATH_* bits of the events' file node), label bool [N] (slot 1 or 2 on the file node).
    node_g: -1 or None = no rename target (a non-merge rename target g is touched like p and f and adds 2 to f's degree)."""
    N = int(n_nodes)
    P = np.asarray(node_p, np.int64); F = np.asarray(node_f, np.int64)
    n = P.shape[0]
    assert n < (1 << 29), "a window holds fewer than 2^29 events"
    Gn = np.full(n, -1, np.int64) if node_g is None else np.asarray(node_g, np.int64)
    t = np.asarray(t, np.float64) + 0.0                      # -0.0 is the time +0.0
    s = np.asarray(slot, np.int64)
    b = clamped(nbytes)
    has_g = Gn >= 0
    for ids in (P, F, Gn[has_g]):
        assert ids.size == 0 or (ids.min() >= 0 and ids.max() < N)
    assert np.all(t >= 0.0) and (s.size == 0 or s.max() <= 7)
    tn = np.concatenate([P, F, Gn[has_g]])
    ts = np.concatenate([s, s, s[has_g]])
    tb = np.concatenate([b, b, b[has_g]])
    tt = np.concatenate([t, t, t[has_g]])
    cnt = np.zeros((N, 8), np.int64)
    np.add.at(cnt, (tn, ts), 1)
    deg = np.zeros(N, np.int64)
    np.add.at(deg, P, 1); np.add.at(deg, F, np.where(has_g, 2, 1)); np.add.at(deg, Gn[has_g], 1)
    bsum = np.zeros(N, np.int64)                             # exact: < 2^29 * 3 events of <= MAX_RW_COUNT bytes < 2^63
    np.add.at(bsum, tn, tb)
    first = np.full(N, np.inf); last = np.full(N, -np.inf)
    np.minimum.at(first, tn, tt); np.maximum.at(last, tn, tt)
    flags = np.zeros(N, np.int64)
    np.bitwise_or.at(flags, F, np.asarray(pflags, np.int64))
    label = np.zeros(N, bool)
    label[F[(s == 1) | (s == 2)]] = True
    return dict(cnt=cnt, deg=deg, bytes=[int(v) for v in bsum.tolist()], first=first, last=last, flags=flags, label=label)


def node_features(node_p, node_f, node_g, t, slot, nbytes, pflags, kind, window):
    """-> x float32 [N, 32], label int32 [N], size_mb float32 [N], acc (node_accumulate's dict).  Every node must be
    touched by an event (interned nodes are)."""
    kind = np.asarray(kind, np.int64)
    N = kind.shape[0]
    a = node_accumulate(node_p, node_f, node_g, t, slot, nbytes, pflags, N)
    assert np.all(np.isfinite(a["first"])), "every node is touched by at least one event"
    f64 = lambda v: np.asarray(v, np.float64)
    x = np.zeros((N, 32), np.float32)
    x[:, 0] = kind == 0
    x[:, 1] = kind == 1
    d = np.log1p(f64(a["deg"])).astype(np.float32)
    x[:, 3] = d; x[:, 4] = d
    x[:, 5:13] = np.log1p(f64(a["cnt"])).astype(np.float32)
    nb = np.asarray([float(v) for v in a["bytes"]], np.float64)      # one rounding of the exact integer sum
    x[:, 13] = (np.log1p(nb) / 20.0).astype(np.float32)
    x[:, 14] = ((a["last"] - a["first"]) / window).astype(np.float32)
    x[:, 15] = (a["first"] / window).astype(np.float32)
    x[:, 16] = (a["flags"] & PATH_LOCKBIT) != 0
    x[:, 17] = (a["flags"] & PATH_NOTE) != 0
    x[:, 18] = (a["flags"] & PATH_TMP) != 0
    wr = f64(a["cnt"][:, 1]) + f64(a["cnt"][:, 5])
    x[:, 19] = np.where(wr > 0, f64(a["cnt"][:, 2]) / np.where(wr > 0, wr, 1.0), 0.0).astype(np.float32)
    k3 = np.maximum(f64(a["cnt"][:, 0]) + f64(a["cnt"][:, 1]) + f64(a["cnt"][:, 2]), 1.0)
    size_mb = np.where(kind == 0, nb / k3 / 1e6, 0.0).astype(np.float32)
    return x, a["label"].astype(np.int32), size_mb, a


def file_sequences(cand, F, t, slot, nbytes, pflags, t0, span, t_max):
    """Per-candidate sequences: the last t_max events (in rank order) whose file node F is the candidate, oldest first.
    Row k: one-hot slot (8), log1p(clamped bytes) / 20, dt to the previous KEPT event clipped at 10 (0 for the first kept
    event), (t - t0) / span, pflags & 1, pflags & 4; zero rows after the length.  t: absolute float64 times by rank.
    -> seq float32 [A, t_max, 16], lengths int32 [A]."""
    F = np.asarray(F, np.int64); t = np.asarray(t, np.float64)
    s = np.asarray(slot, np.int64); b = clamped(nbytes); pf = np.asarray(pflags, np.int64)
    by_file = np.argsort(F, kind="stable")                    # rank order inside each file
    Fs = F[by_file]
    cand = np.asarray(cand, np.int64)
    seq = np.zeros((cand.shape[0], t_max, D_IN), np.float32)
    lengths = np.zeros(cand.shape[0], np.int32)
    lo = np.searchsorted(Fs, cand, "left"); hi = np.searchsorted(Fs, cand, "right")
    for c in range(cand.shape[0]):
        ev = by_file[max(lo[c], hi[c] - t_max):hi[c]]
        L = ev.shape[0]
        lengths[c] = L
        if L == 0:
            continue
        rows = seq[c, :L]
        rows[np.arange(L), s[ev]] = 1.0
        rows[:, 8] = (np.log1p(b[ev].astype(np.float64)) / 20.0).astype(np.float32)
        te = t[ev]
        dt = np.zeros(L)
        dt[1:] = np.minimum(te[1:] - te[:-1], 10.0)
        rows[:, 9] = dt.astype(np.float32)
        rows[:, 10] = ((te - t0) / span).astype(np.float32)
        rows[:, 11] = (pf[ev] & 1) != 0
        rows[:, 12] = (pf[ev] & 4) != 0
    return seq, lengths


def csr_rows(rowptr) -> np.ndarray:
    """the row (destination) of every CSR edge"""
    rowptr = np.asarray(rowptr, np.int64)
    return np.repeat(np.arange(rowptr.shape[0] - 1, dtype=np.int64), np.diff(rowptr))


def edge_labels(node_p, node_f, raw_slot, dst, col):
    """uint8 [E] in CSR order: edge i (src = col[i], dst = dst[i], its row) is 1 iff (src, dst) or (dst, src) is a pair
    (p, f) of an event with raw annotation slot 1..3 (encrypt start / complete, ransom note).  Node kinds play no part."""
    s = np.asarray(raw_slot, np.int64)
    att = (s >= 1) & (s <= 3)
    pairs = set(zip(np.asarray(node_p, np.int64)[att].tolist(), np.asarray(node_f, np.int64)[att].tolist()))
    return np.asarray([(a, d) in pairs or (d, a) in pairs
                       for a, d in zip(np.asarray(col, np.int64).tolist(), np.asarray(dst, np.int64).tolist())], np.uint8)
