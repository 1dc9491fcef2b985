"""The window-graph kernels of csrc/graph.cu and csrc/intern_device.cu -- per-node features, per-file LSTM sequences,
per-pair edge labels, interning and name / directory hashes -- against the exact statement oracle/window_ref.py (itself
held to the event-by-event spec in test_window_statement_cpu.py) and the host interning, at the shapes where they change
over: byte counts from the whole uint64 range, 2^24+ counts on one atomic, truncated sequences, candidate counts around
the 8 warps of a block, int64 rowptr, 1 / 2 / 7 / 8 radix passes for the pair keys, file-table growth, long rename chains.

Tolerances: everything derived from integers or flags, the time columns (one double expression, rounded once), size_mb,
lengths, labels, ids and hashes bit for bit; the log1p columns within 1 fp32 ulp (CUDA's and numpy's double log1p may
differ in the last bit of the double, which survives the rounding to fp32 only at a tie); every value finite."""
import ctypes as C

import numpy as np
import pytest
import torch

from nerrf_b200 import _lib, graph as G, ingest, stream
from nerrf_b200._lib import NerrfError
from nerrf_b200.ai.models import lstm
from oracle import window_ref as W

pytestmark = pytest.mark.gpu

BYTE_EDGES = (0, 1, 0x7ffff000, 0x7ffff001, 2 ** 63 - 1, 2 ** 63, 2 ** 64 - 1)
LOG_COLS = list(range(3, 14))                     # degree, the eight counts, bytes
EXACT_COLS = [c for c in range(32) if c not in LOG_COLS]


def cu(a, dt):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a).astype(dt, copy=False))).cuda()


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def assert_ulp1(got, want):
    assert np.all(np.isfinite(got)), np.argwhere(~np.isfinite(got))[:5]
    bad = np.abs(got.astype(np.float64) - want) > np.spacing(np.abs(want)).astype(np.float64)
    assert not bad.any(), (np.argwhere(bad)[:5], got[bad][:5], want[bad][:5])


# ------------------------------------------------------------------------------------------------ per-node features
def check_features(P, F, Gn, t, slot, nbytes, pf, kind, window=60.0):
    nb = np.asarray(nbytes, np.uint64).view(np.int64)                    # the wire's bits, as DeviceStream holds them
    x, label, size_mb = G.node_features_device(cu(P, np.int32), cu(F, np.int32), None if Gn is None else cu(Gn, np.int32),
                                               cu(t, np.float64), cu(slot, np.uint8), cu(nb, np.int64), cu(pf, np.uint8),
                                               cu(kind, np.int8), window)
    x, label, size_mb = x.cpu().numpy(), label.cpu().numpy(), size_mb.cpu().numpy()
    wx, wlabel, wsize, acc = W.node_features(P, F, Gn, t, slot, np.asarray(nbytes, np.uint64), pf, kind, window)
    assert np.all(np.isfinite(x)) and np.all(np.isfinite(size_mb))
    assert np.array_equal(bits(x[:, EXACT_COLS]), bits(wx[:, EXACT_COLS])), np.argwhere(x[:, EXACT_COLS] != wx[:, EXACT_COLS])[:5]
    assert_ulp1(x[:, LOG_COLS], wx[:, LOG_COLS])
    assert np.array_equal(bits(size_mb), bits(wsize)), (size_mb[size_mb != wsize][:5], wsize[size_mb != wsize][:5])
    assert np.array_equal(label, wlabel)
    return x, size_mb, acc


def test_node_features_byte_counts_from_the_whole_uint64_range():
    # node 0: the process; file 1 + k: one write of BYTE_EDGES[k] alone; file 8: all of them plus 100 bytes; file 9: a
    # 2^64 - 1 write and a 100-byte write (a uint64 sum wraps to 99); file 10: 64 writes of 2^64 - 1
    vals = list(BYTE_EDGES) + list(BYTE_EDGES) + [100, 2 ** 64 - 1, 100] + [2 ** 64 - 1] * 64
    F = list(range(1, 8)) + [8] * 8 + [9, 9] + [10] * 64
    n = len(F)
    P = np.zeros(n, np.int64); t = np.linspace(0.0, 30.0, n)
    slot = np.full(n, 5); pf = np.zeros(n)
    kind = np.r_[1, np.zeros(10)]
    x, size_mb, acc = check_features(P, np.asarray(F), None, t, slot, vals, pf, kind)
    cap = G.MAX_RW_COUNT
    assert acc["bytes"][9] == cap + 100 and acc["bytes"][10] == 64 * cap
    assert acc["bytes"][0] == sum(min(v, cap) for v in vals)
    assert size_mb[9] == np.float32((cap + 100) / 1e6)                   # writes are slot 5: k = 1


def test_node_features_contention_and_counts_above_2_24():
    # one pid in every event (2^24 + 1000 same-address atomics), so its slot-5 count passes 2^24 where fp32 stops being exact
    rng = np.random.default_rng(1)
    n = (1 << 24) + 1000
    N = 64
    P = np.zeros(n, np.int64)
    F = rng.integers(1, N, n)
    slot = np.full(n, 5)
    slot[rng.integers(0, n, 500)] = rng.integers(0, 8, 500)
    nbytes = np.where(rng.random(n) < 1e-4, np.uint64(2 ** 64 - 1), rng.integers(0, 1 << 16, n).astype(np.uint64))
    t = np.sort(rng.random(n) * 60.0)
    pf = rng.integers(0, 16, n)
    kind = np.r_[1, np.zeros(N - 1)]
    _, _, acc = check_features(P, F, None, t, slot, nbytes, pf, kind)
    assert acc["cnt"][0, 5] > (1 << 24) and acc["deg"][0] == n


def test_node_features_renames_times_ratios_slot7_and_labels():
    # node 0, 1: processes; 2..9: files.  Non-merge renames with g == f (f's degree + 3 for that event) and g != f;
    # t = 0, t = -0.0 and a node touched once (first == last); a file with only completes (wr = 0); slot 7; slot 3 on a
    # file (a ransom note: no label), slots 1 and 2 label their file
    P = [0, 0, 1, 1, 0, 1, 0, 1, 0, 1]
    F = [2, 2, 3, 4, 5, 6, 7, 8, 9, 9]
    Gn = [2, -1, 4, -1, -1, 5, -1, -1, -1, -1]
    t = [-0.0, 0.0, 0.0, 1.5, 2.0, 7.25, 7.25, 9.0, 59.9, 60.0]
    slot = [6, 6, 6, 2, 2, 7, 1, 3, 0, 4]
    pf = [1, 0, 4, 2, 0, 1, 8, 2, 4, 0]
    nbytes = [0, 2 ** 64 - 1, 5, 2 ** 63, 7, 0, 1, 0x7ffff001, 3, 0]
    kind = [1, 1] + [0] * 8
    x, _, acc = check_features(*(np.asarray(a) for a in (P, F, Gn, t, slot, nbytes, pf, kind)))
    assert acc["deg"][2] == 3 + 1 and acc["label"][5] and acc["label"][7] and not acc["label"][8]
    assert x[4, 19] == 0.0 and x[2, 15] == 0.0 and not np.signbit(x[2, 15])
    rng = np.random.default_rng(2)                         # and the same kinds of events at random, 3 event slots of each
    n, N = 50_000, 3000
    P = rng.integers(0, 100, n); F = rng.integers(100, N, n)
    Gn = np.where(rng.random(n) < 0.2, np.where(rng.random(n) < 0.5, F, rng.integers(100, N, n)), -1)
    t = np.sort(rng.integers(0, 600, n) * 0.1); t[:5] = -0.0
    slot = rng.integers(0, 8, n); pf = rng.integers(0, 16, n)
    nbytes = np.asarray(BYTE_EDGES, np.uint64)[rng.integers(0, len(BYTE_EDGES), n)]
    touched = np.zeros(N, bool); touched[P] = touched[F] = True; touched[Gn[Gn >= 0]] = True
    keep = touched[np.arange(N)]
    remap = np.cumsum(keep) - 1                            # every node touched (interned nodes are)
    kind = np.r_[np.ones(100), np.zeros(N - 100)][keep]
    Gr = np.where(Gn >= 0, remap[np.maximum(Gn, 0)], -1)
    check_features(remap[P], remap[F], Gr, t, slot, nbytes, pf, kind, window=37.5)


# ------------------------------------------------------------------------------------------------ sequences
def _seq_events(degrees, seed):
    """file k gets degrees[k] events: equal timestamps inside a file, gaps of exactly 10 s and above, byte counts from
    BYTE_EDGES, paths with .lockbit / /tmp flags, several pids"""
    rng = np.random.default_rng(seed)
    ev = []
    for k, d in enumerate(degrees):
        sec, nan = 1_700_000_000, 0
        base = ["/tmp/s%d" % k, "/srv/s%d" % k][k % 2]
        for i in range(d):
            step = int(rng.choice([0, 0, 1, 10, 11, 25]))
            sec += step
            path = base + [".dat", ".lockbit3", ".x"][int(rng.integers(3))]
            ev.append({"ts": (sec, nan), "pid": int(rng.integers(1, 5)), "syscall": ["openat", "write", "rename", "unlink"][int(rng.integers(4))],
                       "path": path, "bytes": int(rng.choice(BYTE_EDGES)) if rng.random() < 0.5 else int(rng.integers(0, 4096))})
    return ingest.decode_event_batch(ingest.encode_event_batch(ev))


def _stream_statement(ds, g):
    """the statement's per-rank columns of window graph g of DeviceStream ds (node ids from the device interning)"""
    lo, hi = g.meta["window_ranks"]
    order = ds.order[lo:hi]
    F = ds.node_f[ds.d_order[lo:hi]].cpu().numpy()
    slot = np.asarray(G.OBSERVABLE_SLOT, np.int64)[ds.cols.event_slot[order]]
    return dict(F=F, t=ds.ts_sorted[lo:hi], slot=slot, bytes=ds.cols.bytes[order], pf=ds.cols.path_flags[order],
                t0=g.meta["t0"], span=g.meta["span"])


def check_sequences(seq, ln, cand, s, t_max):
    seq, ln = seq.cpu().numpy(), ln.cpu().numpy()
    wseq, wln = W.file_sequences(cand, s["F"], s["t"], s["slot"], s["bytes"], s["pf"], s["t0"], s["span"], t_max)
    assert np.array_equal(ln, wln)
    assert np.all(np.isfinite(seq))
    other = [c for c in range(16) if c != 8]
    assert np.array_equal(bits(seq[:, :, other]), bits(wseq[:, :, other]))
    assert_ulp1(seq[:, :, 8], wseq[:, :, 8])


DEGREES = [1, 31, 32, 33, 99, 100, 101, 5000]


@pytest.fixture(scope="module")
def seq_window():
    cols = _seq_events(DEGREES, 3)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    g = ds.window_graph(t0 - 1, t1, 60.0)
    return ds, g, _stream_statement(ds, g)


@pytest.mark.parametrize("n_cand", [1, 7, 8, 9, 4097])
def test_sequences_device_against_the_statement(seq_window, n_cand):
    ds, g, s = seq_window
    files = np.nonzero(g.meta["node_kind"] == 0)[0]
    assert sorted(np.bincount(s["F"])[files].tolist()) == sorted(DEGREES)
    rng = np.random.default_rng(n_cand)
    cand = rng.choice(files, n_cand, replace=True)                       # duplicates, any order
    if n_cand >= len(files):
        cand[:len(files)] = rng.permutation(files)                       # every degree at least once
    seq, ln = ds.sequences_device(g, cand)
    check_sequences(seq, ln, cand, s, lstm.T_MAX)
    if n_cand == 4097:
        assert set(ln.cpu().numpy().tolist()) == {min(d, lstm.T_MAX) for d in DEGREES}


def _sequences_direct(ds, g, cand, rowptr, perm, t_max):
    A = len(cand)
    cand_d = cu(cand, np.int64)
    seq = torch.empty(A, t_max, lstm.D_IN, dtype=torch.float32, device="cuda")
    ln = torch.empty(A, dtype=torch.int32, device="cuda")
    lo, hi = g.meta["window_ranks"]
    _lib.check(_lib.lib().nerrf_trace_sequences(_lib.ptr(cand_d), A, _lib.ptr(rowptr), int(rowptr.dtype == torch.int64), _lib.ptr(perm),
                                                _lib.ptr(ds.d_order[lo:hi]), _lib.ptr(ds.d_ts), _lib.ptr(ds.d_slot), _lib.ptr(ds.d_bytes),
                                                _lib.ptr(ds.d_pf_raw), float(g.meta["t0"]), float(g.meta["span"]), t_max, _lib.ptr(seq),
                                                _lib.ptr(ln), _lib.current_stream_ptr()), "nerrf_trace_sequences")
    return seq, ln


@pytest.mark.parametrize("t_max", [1, 33, lstm.T_MAX])
def test_sequences_kernel_int64_rowptr_empty_rows_and_t_max(seq_window, t_max):
    # the window's CSR rebuilt with one extra node (an empty last row) and an int64 rowptr: a candidate of degree 0 has
    # length 0 and zero rows
    ds, g, s = seq_window
    N = g.num_nodes
    lo, hi = g.meta["window_ranks"]
    sel = ds.d_order[lo:hi]
    P, F = ds.node_p[sel], ds.node_f[sel]
    src = torch.stack([P, F], 1).reshape(-1).contiguous(); dst = torch.stack([F, P], 1).reshape(-1).contiguous()
    te = (ds.d_ts[sel] - g.meta["t0"]).to(torch.float32).repeat_interleave(2).contiguous()
    rowptr, col, _, perm = G.build_csr_device(src, dst, te, torch.ones_like(te), N + 1, t_ref=float(g.meta["span"]),
                                              rowptr_dtype=torch.int64, return_perm=True)
    assert torch.equal(rowptr[:-1].to(g.rowptr.dtype), g.rowptr) and int(rowptr[-1] - rowptr[-2]) == 0
    files = np.nonzero(g.meta["node_kind"] == 0)[0]
    cand = np.r_[N, files, files[::-1], N]
    seq, ln = _sequences_direct(ds, g, cand, rowptr, perm, t_max)
    check_sequences(seq, ln, cand, s, t_max)
    assert int(ln[0]) == 0 and not bool(seq[0].any())


def test_sequences_device_refuses_candidates_outside_the_graph(seq_window):
    ds, g, _ = seq_window
    for bad in ([g.num_nodes], [0, -1], [1, 2, g.num_nodes + 100]):
        with pytest.raises(NerrfError, match="candidate"):
            ds.sequences_device(g, bad)


# ------------------------------------------------------------------------------------------------ edge labels
def _labels(P, F, raw, dst, col, N, rowptr):
    got = G.edge_labels_device(cu(P, np.int32), cu(F, np.int32), cu(raw, np.uint8), rowptr, cu(col, np.int32), N).cpu().numpy()
    want = W.edge_labels(P, F, raw, dst, col)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    return got


@pytest.mark.parametrize("N", [1, 15, 16])
@pytest.mark.parametrize("E", [1, 255, 256, 257])
def test_edge_labels_small_graphs(N, E):
    # 15 nodes: pair keys below 2^8 (one radix pass, the result in the other buffer); 16: 2^8 needs 9 bits (two passes)
    rng = np.random.default_rng(N * 1000 + E)
    n = 300
    P = rng.integers(0, N, n); F = rng.integers(0, N, n)
    raw = rng.integers(0, 8, n)
    raw[:40] = 2; P[40:60] = P[:20]; F[40:60] = F[:20]; raw[40:60] = 1       # duplicate attack events
    lo_row, hi_row = (1, N - 1) if N >= 3 else (0, N)                        # empty first and last rows
    pool_src = np.r_[P, F, rng.integers(0, N, n)]
    pool_dst = np.r_[F, P, rng.integers(0, N, n)]                            # both orientations, plus unrelated links
    ok = (pool_dst >= lo_row) & (pool_dst < hi_row)
    pool_src, pool_dst = pool_src[ok], pool_dst[ok]
    pick = rng.integers(0, pool_src.shape[0], E)
    src, dst = pool_src[pick], pool_dst[pick]
    rowptr, col, _ = G.build_csr_device(cu(src, np.int32), cu(dst, np.int32), cu(np.zeros(E), np.float32), cu(np.ones(E), np.float32), N)
    rp = rowptr.cpu().numpy()
    if N >= 3:
        assert rp[1] == 0 and rp[N - 1] == rp[N] == E
    lab = _labels(P, F, raw, W.csr_rows(rp), col.cpu().numpy(), N, rowptr)
    if E >= 255 and N > 1:
        assert lab.any() and not lab.all()


@pytest.mark.parametrize("N", [(1 << 28) - 1, (1 << 28) + 1])
def test_edge_labels_near_2_28_nodes(N):
    # pair keys of 56 / 57 bits: 7 / 8 radix passes; a few events on ids near N - 1; rowptr of 2^28 rows built in place
    ids = [0, 1, N - 3, N - 2, N - 1]
    P = np.asarray([N - 1, N - 2, 0, N - 1, 1, N - 3, N - 1, N - 2])
    F = np.asarray([N - 2, N - 1, N - 1, N - 3, 0, 1, 0, N - 1])
    raw = np.asarray([1, 0, 3, 2, 5, 1, 4, 2])
    src, dst = [], []
    for p, f in zip(P.tolist(), F.tolist()):
        src += [p, f]; dst += [f, p]
    src += [N - 3, N - 2]; dst += [N - 2, N - 3]                             # a file <-> file link of no attack event
    o = np.lexsort((src, dst))
    src, dst = np.asarray(src)[o], np.asarray(dst)[o]
    rowptr = torch.zeros(N + 1, dtype=torch.int32, device="cuda")
    for v, c in zip(*np.unique(dst, return_counts=True)):
        rowptr[int(v) + 1:] += int(c)
    lab = _labels(P, F, raw, dst, src, N, rowptr)
    assert lab.any() and int(rowptr[-1]) == len(src) and set(ids) >= set(dst.tolist())
    del rowptr
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ interning and hashes
def _same_interning(cols, merge=True):
    order = np.argsort(cols.timestamp, kind="stable")
    want = ingest.intern_nodes(cols, order, merge)
    got = ingest.intern_nodes_device(cols, order, merge)
    for name, a, b in zip(("node_p", "node_f", "node_g", "kind", "name_event", "name_which"), got, want):
        assert np.array_equal(a, b), name
    return want


def _hashes_match(cols):
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    g = ds.window_graph(t0 - 1, t1, 60.0)
    names = [g.meta["names"][v] for v in range(g.num_nodes)]
    nh, dh = g.meta["name_hash"].cpu().numpy(), g.meta["dir_hash"]().cpu().numpy()
    assert nh.tolist() == [stream.name_hash(s) for s in names]
    assert dh.tolist() == [stream.dir_hash(s) for s in names]
    return g


def _ev(t, pid, path, new_path=""):
    return {"ts": (1_700_000_000 + t, 0), "pid": pid, "syscall": "rename" if new_path else "openat", "path": path, "new_path": new_path}


@pytest.mark.parametrize("L", [1, 2, 63, 4096])
def test_interning_merge_rename_chains(L):
    # /c/f0 -> /c/f1 -> ... -> /c/fL: one node for the whole chain (root_of walks it), named by the last name
    ev = [_ev(0, 5, "/c/f0.dat")] + [_ev(1 + i, 5, "/c/f%d.dat" % i, "/c/f%d.dat" % (i + 1)) for i in range(L)]
    ev.append(_ev(L + 2, 6, "/c/f%d.dat" % L))
    cols = ingest.decode_event_batch(ingest.encode_event_batch(ev))
    node_p, node_f, _, kind, _, _ = _same_interning(cols)
    assert len(set(node_f.tolist())) == 1 and kind.shape[0] == 3
    _hashes_match(cols)


@pytest.mark.parametrize("n", [256, 257])
@pytest.mark.parametrize("merge", [True, False])
def test_interning_every_event_a_new_path_and_target(n, merge):
    # the largest table load: two new keys per event (the file table grows from 1024 to 2048 slots between 256 and 257)
    ev = [_ev(i, 1000 + i, "/n/a%d.dat" % i, "/n/b%d.x" % i) for i in range(n)]
    cols = ingest.decode_event_batch(ingest.encode_event_batch(ev))
    want = _same_interning(cols, merge)
    assert want[3].shape[0] == (2 * n if merge else 3 * n)
    if merge:
        _hashes_match(cols)


def test_interning_odd_and_long_paths():
    long_a = "/" + "a" * 69_999
    long_b = "/d/" + "b.c" * 23_333 + "/e"
    paths = ["x", "/x", "/a/b/", "/a/b.c.d", long_a, long_b, "/a/b.c", "/a/b", long_a + ".z"]
    ev = [_ev(i, 1 + i % 3, p) for i, p in enumerate(paths)]
    ev += [_ev(20, 1, "/a/b.c.d", "/a/b/"), _ev(21, 2, long_b, long_a + ".q"), _ev(22, 3, "x", "y.z")]
    cols = ingest.decode_event_batch(ingest.encode_event_batch(ev))
    assert int(np.diff(cols.strings["path"][0]).max()) >= 70_000
    for merge in (True, False):
        _same_interning(cols, merge)
    g = _hashes_match(cols)
    names = {g.meta["names"][v] for v in range(g.num_nodes)}
    assert long_a in names or long_a + ".z" in names or long_a + ".q" in names


def test_empty_paths_resolve_to_the_open_file():
    # "" is a path only for an event that names nothing: resolve_columns gives it the pid's open file, or drops it
    ev = [_ev(0, 1, ""), _ev(1, 2, "/k/a"), _ev(2, 2, "")]
    cols = ingest.resolve_columns(ingest.decode_event_batch(ingest.encode_event_batch(ev)))
    assert cols.n == 2
    _same_interning(cols)
    _hashes_match(cols)


# ------------------------------------------------------------------------------------------------ scale
@pytest.fixture(scope="module")
def models():
    from nerrf_b200.ai import train as T
    from nerrf_b200.ai.models import GraphSAGE_T
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), lstm.LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3)
    return model.cuda(), scorer.cuda()


def test_fleet_window_with_injected_huge_writes(models):
    cols, enc, bad = stream.fleet_columns(9700, 24, seed=5, return_pids=True)
    assert cols.n >= 1_000_000
    attacker = np.isin(cols.pid, [int(s[4:]) for s in bad])
    writes = np.nonzero(attacker & ((cols.event_slot == 5) | (cols.event_slot == 1)))[0]
    inj = writes[np.random.default_rng(0).choice(writes.shape[0], 6, replace=False)]
    hot = ingest.EventColumns(**{**cols.__dict__, "bytes": cols.bytes.copy()})
    hot.bytes[inj] = np.uint64(2 ** 64 - 1)

    ds = stream.DeviceStream(hot, "cuda", observable=True)
    t0, t1 = ds.span()
    g = ds.window_graph(t0 - 1, t1, 60.0)
    lo, hi = g.meta["window_ranks"]
    assert hi - lo >= 1_000_000
    sel = ds.d_order[lo:hi]
    order = ds.order[lo:hi]
    Pw, Fw = ds.node_p[sel].cpu().numpy(), ds.node_f[sel].cpu().numpy()
    pf = ds.d_pf[sel].cpu().numpy()
    slot = np.asarray(G.OBSERVABLE_SLOT, np.int64)[ds.cols.event_slot[order]]
    wx, _, wsize, _ = W.node_features(Pw, Fw, None, ds.ts_sorted[lo:hi] - g.meta["t0"], slot, ds.cols.bytes[order], pf,
                                      g.meta["node_kind"], 60.0)
    x = g.x.cpu().numpy()
    assert np.all(np.isfinite(x))
    assert np.array_equal(bits(x[:, EXACT_COLS]), bits(wx[:, EXACT_COLS]))
    assert_ulp1(x[:, LOG_COLS], wx[:, LOG_COLS])
    assert np.array_equal(bits(g.meta["size_mb"]), bits(wsize))
    hit = np.unique(Fw[ds.cols.bytes[order] == np.uint64(2 ** 64 - 1)])
    assert hit.size and np.all(wsize[hit] > 0)
    s = _stream_statement(ds, g)
    files = np.nonzero(g.meta["node_kind"] == 0)[0]
    top = np.r_[hit, np.random.default_rng(1).choice(files, 4096 - hit.size, replace=False)]
    seq, ln = ds.sequences_device(g, top)
    check_sequences(seq, ln, top, s, lstm.T_MAX)

    # the planner over the same trace with and without the huge writes: a clamped 2 GB write is a real feature change
    # (bytes column, action size), so the two plans need not be identical, but both must still find the attack
    model, scorer = models
    for c in (cols, hot):
        sp = stream.StreamingPlanner(model, scorer, top_a=1024, n_rollouts=512, depth=24, iterations=8, commit_per_search=32,
                                     kill_candidates=True)
        sp.run(c)
        planned = set(sp.reverted)
        assert len(planned & enc) >= 0.90 * len(enc) and len(planned & enc) >= 0.90 * len(planned)
        assert sp.killed and set(sp.killed) <= bad
