"""The GraphSAGE-T layer backward (csrc/sage_bwd.cu) at stream-window scale, on degenerate graphs, and from run to run
(needs an H100 except the workspace sweep).

The dW reduction splits the rows into at most MAX_CHUNKS = 264 chunks of whole 32-row tiles, so the node counts below are
chosen against that cap: up to 8448 nodes every chunk is one tile; 8449 is one tile more than the cap; 100 003 gives 261
chunks of 384 rows with a partial last chunk and a partial last tile; 300 007 gives 261 chunks of 1152 rows.  Every
gradient is compared with the float64 oracle's sparse path (oracle/sage_bwd_ref.py, tests/edge_head_ref.py) under the
bound of tests/test_gpu_train.py, |got - want| <= 2e-4 |want| + 2e-5 rms(want); the worst error ratio against that
bound is printed per tensor."""
import ctypes as C

import numpy as np
import pytest
import torch

from edge_head_ref import model_backward_with_edges
from nerrf_b200 import _lib as L, graph as G
from nerrf_b200.ai import autograd as AG
from nerrf_b200.ai.models import GraphSAGE_T
from oracle import sage_bwd_ref as B

RTOL, ATOL_RMS = 2e-4, 2e-5
HB, DW_BR, MAX_CHUNKS = 128, 32, 264
gpu = pytest.mark.gpu


def _plan(n):
    """(chunks, rows per chunk) of the dW reduction: a function of n alone."""
    tiles = max(1, -(-n // DW_BR))
    c = min(tiles, MAX_CHUNKS)
    rpc = -(-tiles // c) * DW_BR
    return max(1, -(-n // rpc)), rpc


def _workspace_bytes(n, F):
    chunks, _ = _plan(n)
    return ((n * 2 * F * 4 + 255) & ~255) + chunks * 2 * F * HB * 4 + chunks * HB * 4 + 256


def _ratio(got, want):
    """max |got - want| / (RTOL |want| + ATOL_RMS rms(want)): <= 1 is inside the bound."""
    got = np.asarray(got.detach().double().cpu().numpy() if hasattr(got, "detach") else got, np.float64)
    want = np.asarray(want, np.float64)
    assert got.shape == want.shape
    if want.size == 0:
        return 0.0
    rms = float(np.sqrt((want ** 2).mean()))
    return float((np.abs(got - want) / (RTOL * np.abs(want) + ATOL_RMS * max(rms, 1e-30))).max())


def _graph(N, E, kind, seed):
    """(rowptr int32, col, ew): synthetic_graph with hub sources / hub destinations, or oracle degenerate_graph."""
    if kind == "degenerate":
        return B.degenerate_graph(N, E, seed)
    g = G.synthetic_graph(N=N, E=E, seed=seed, hub=kind, f_in=32)
    return g.rowptr, g.col, g.ew


def _train_graph(rowptr, col, ew, rp64):
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return AG.TrainGraph(c(rowptr.astype(np.int64 if rp64 else np.int32)), c(col), c(ew))


def _layer_bwd(tg, h, m, y, dy, W, F, dh=True, dw=True, relu=1):
    """One nerrf_sage_layer_bwd call; the tensors a part does not need are passed as NULL."""
    n = tg.n
    out_dh = torch.empty(n, F, device="cuda") if dh else None
    dW = torch.empty(2 * F, HB, device="cuda") if dw else None
    db = torch.empty(HB, device="cuda") if dw else None
    need = C.c_size_t()
    L.check(L.lib().nerrf_sage_layer_bwd_workspace_bytes(n, F, C.byref(need)), "workspace_bytes")
    ws = torch.empty((need.value + 3) // 4, device="cuda")
    L.check(L.lib().nerrf_sage_layer_bwd(L.ptr(h if dw else None), L.ptr(m if dw else None), L.ptr(y if relu else None),
                                         L.ptr(dy), L.ptr(W), L.ptr(tg.t_rowptr), int(tg.t_rowptr.dtype == torch.int64),
                                         L.ptr(tg.t_col), L.ptr(tg.t_w), L.ptr(out_dh), L.ptr(dW), L.ptr(db), L.ptr(ws),
                                         need.value, n, F, HB, relu, L.current_stream_ptr()), "nerrf_sage_layer_bwd")
    torch.cuda.synchronize()
    return out_dh, dW, db


# ------------------------------------------------------------------------------------ (a) one layer through the ABI
LAYER_CASES = [  # N, E, F, graph, int64 rowptr
    (8448, 80_000, 32, "src", False),
    (8449, 80_000, 64, "dst", True),
    (8449, 60_000, 128, "degenerate", False),
    (100_003, 1_000_000, 128, "dst", False),
    (100_003, 1_000_000, 32, "src", True),
    (100_003, 600_000, 64, "degenerate", True),
    (300_007, 2_000_000, 64, "dst", True),
    (300_007, 2_000_000, 128, "src", False),
    (5000, 0, 32, "degenerate", False),
    (5000, 0, 128, "degenerate", True),
]


@gpu
@pytest.mark.parametrize("N,E,F,kind,rp64", LAYER_CASES)
def test_layer_backward_at_scale_matches_the_float64_statement(N, E, F, kind, rp64):
    """h random non-negative, y = the device forward's output, m = the standalone aggregate of h, dy random; the fp64
    statement is evaluated at the device's y, so the ReLU mask is the kernel's own.  dh-only and dW-only calls give the
    bits of the combined call."""
    rowptr, col, ew = _graph(N, E, kind, seed=N + F)
    tg = _train_graph(rowptr, col, ew, rp64)
    rng = np.random.default_rng(N + E + F)
    h = torch.from_numpy(np.maximum(rng.standard_normal((N, F)), 0).astype(np.float32)).cuda()
    model = GraphSAGE_T(F, HB, 1, seed=F).cuda()
    W = model.weights[0].detach().contiguous()
    with torch.no_grad():
        y = model.layer_forward(0, h, tg.rowptr, tg.col, tg.edge_w)
    m = AG.aggregate(h, tg)
    dy = torch.from_numpy(rng.standard_normal((N, HB)).astype(np.float32)).cuda()
    dh, dW, db = _layer_bwd(tg, h, m, y, dy, W, F)
    hn = h.cpu().numpy()
    want_m = B.aggregate(hn, rowptr, col, ew, sparse=True)
    want = B.layer_backward(hn, want_m, y.cpu().numpy(), dy.cpu().numpy(), W.cpu().numpy(), rowptr, col, ew, sparse=True)
    ratios = {k: _ratio(g, w) for k, g, w in zip(("dh", "dW", "db"), (dh, dW, db), want)}
    chunks, rpc = _plan(N)
    deg_in = np.diff(rowptr.astype(np.int64))
    print(f"N={N} E={col.size} F={F} {kind} max in-degree {deg_in.max() if N else 0}: {chunks} chunks x {rpc} rows; "
          + ", ".join(f"{k} {r:.3f}" for k, r in ratios.items()))
    for k, r in ratios.items():
        assert r <= 1.0, f"{k}: error ratio {r:.3f} (N={N} F={F} {kind})"
    dh1, none_w, none_b = _layer_bwd(tg, h, m, y, dy, W, F, dw=False)
    none_h, dW1, db1 = _layer_bwd(tg, h, m, y, dy, W, F, dh=False)
    assert none_w is None and none_b is None and none_h is None
    assert torch.equal(dh, dh1) and torch.equal(dW, dW1) and torch.equal(db, db1)


@gpu
def test_layer_backward_without_relu_takes_no_output():
    N, F = 8449, 64
    rowptr, col, ew = _graph(N, 70_000, "dst", seed=5)
    tg = _train_graph(rowptr, col, ew, False)
    rng = np.random.default_rng(5)
    h = torch.from_numpy(np.maximum(rng.standard_normal((N, F)), 0).astype(np.float32)).cuda()
    W = GraphSAGE_T(F, HB, 1, seed=5).weights[0].detach().cuda().contiguous()
    m = AG.aggregate(h, tg)
    dy = torch.from_numpy(rng.standard_normal((N, HB)).astype(np.float32)).cuda()
    dh, dW, db = _layer_bwd(tg, h, m, None, dy, W, F, relu=0)
    hn = h.cpu().numpy()
    want = B.layer_backward(hn, B.aggregate(hn, rowptr, col, ew, sparse=True), np.zeros((N, HB)), dy.cpu().numpy(),
                            W.cpu().numpy(), rowptr, col, ew, relu=False, sparse=True)
    for k, g, w in zip(("dh", "dW", "db"), (dh, dW, db), want):
        assert _ratio(g, w) <= 1.0, k


@gpu
def test_layer_backward_abi_edges():
    """n_nodes = 0 zeroes dW and db; a workspace one byte short is NERRF_ERR_WORKSPACE; a misaligned buffer is refused
    with an error naming the alignment."""
    lib = L.lib()
    F = 64
    buf = torch.zeros(1 << 16, device="cuda")
    t_rowptr = torch.zeros(1, dtype=torch.int32, device="cuda")
    dW = torch.full((2 * F, HB), float("nan"), device="cuda")
    db = torch.full((HB,), float("nan"), device="cuda")
    need = C.c_size_t()
    assert lib.nerrf_sage_layer_bwd_workspace_bytes(0, F, C.byref(need)) == 0 and need.value == _workspace_bytes(0, F)
    ws = torch.empty((need.value + 3) // 4, device="cuda")
    L.check(lib.nerrf_sage_layer_bwd(L.ptr(buf), L.ptr(buf), L.ptr(buf), L.ptr(buf), L.ptr(buf), L.ptr(t_rowptr), 0, None,
                                     None, None, L.ptr(dW), L.ptr(db), L.ptr(ws), need.value, 0, F, HB, 1,
                                     L.current_stream_ptr()), "nerrf_sage_layer_bwd(n_nodes=0)")
    torch.cuda.synchronize()
    assert int(torch.count_nonzero(dW)) == 0 and int(torch.count_nonzero(db)) == 0
    # a real 300-node layer: one byte short of the workspace, then a misaligned dy
    n = 300
    tg = _train_graph(*_graph(n, 3000, "src", seed=1), False)
    h, y, dy = torch.rand(n, F, device="cuda"), torch.rand(n, HB, device="cuda"), torch.rand(n, HB, device="cuda")
    W = torch.rand(2 * F, HB, device="cuda")
    dh = torch.empty(n, F, device="cuda")
    assert lib.nerrf_sage_layer_bwd_workspace_bytes(n, F, C.byref(need)) == 0 and need.value == _workspace_bytes(n, F)
    ws = torch.empty((need.value + 3) // 4, device="cuda")
    call = lambda dy_p, ws_bytes: lib.nerrf_sage_layer_bwd(L.ptr(h), L.ptr(h), L.ptr(y), dy_p, L.ptr(W), L.ptr(tg.t_rowptr),
                                                          0, L.ptr(tg.t_col), L.ptr(tg.t_w), L.ptr(dh), L.ptr(dW),
                                                          L.ptr(db), L.ptr(ws), ws_bytes, n, F, HB, 1,
                                                          L.current_stream_ptr())
    assert call(L.ptr(dy), need.value - 1) == -4                  # NERRF_ERR_WORKSPACE
    assert b"workspace" in lib.nerrf_last_error()
    assert call(C.c_void_p(dy.data_ptr() + 4), need.value) == -1
    assert b"16-byte aligned" in lib.nerrf_last_error()
    assert call(L.ptr(dy), need.value) == 0
    torch.cuda.synchronize()


# -------------------------------------------------------------------------------------- (b) the whole model at scale
def _check_model(model, x, tg, rowptr, col, ew, seed, what):
    """Node and edge losses through AG.sage_logits against the float64 statement evaluated at the device forward's layer
    outputs (the ReLU masks are the device's, as in the single-layer test).  The device outputs themselves are checked
    against the float64 forward (the forward's bound, 1e-4 |y| + 1e-5 rms), and the masks that differ from the float64
    forward's are counted: each one moves the gradient by a whole dy entry, which the gradient bound is not meant to
    absorb once a graph has 10^7+ activations."""
    N, E = x.shape[0], col.size
    rng = np.random.default_rng(seed)
    dlogit = rng.standard_normal(N).astype(np.float32)
    dedge = rng.standard_normal((E, 2)).astype(np.float32)
    acts, h = [], x
    with torch.no_grad():
        for l in range(len(model.weights)):
            h = model.layer_forward(l, h, tg.rowptr, tg.col, tg.edge_w)
            acts.append(h.cpu().numpy())
    x = x.detach().requires_grad_()
    nl, el = AG.sage_logits(model, x, tg)
    ((nl * torch.from_numpy(dlogit).cuda()).sum() + (el * torch.from_numpy(dedge).cuda()).sum()).backward()
    got = {"x": x.grad, "node_w": model.node_w.grad, "node_b": model.node_b.grad, "edge_W": model.edge_W.grad,
           "edge_b": model.edge_b.grad}
    for l, (W, b) in enumerate(zip(model.weights, model.biases)):
        got[f"dW[{l}]"], got[f"db[{l}]"] = W.grad, b.grad
    P, xn = model.oracle_params(), x.detach().cpu().numpy()
    want = model_backward_with_edges(P, xn, rowptr, col, ew, dlogit, dedge, sparse=True, acts=acts)
    for l in range(len(model.weights)):
        want[f"dW[{l}]"], want[f"db[{l}]"] = want["layers"][l]
    flips, hn = [], xn.astype(np.float64)
    for l, (W, b) in enumerate(P["layers"]):
        hn, _ = B.layer_forward(hn, rowptr, col, ew, W, b, sparse=True)
        rms = float(np.sqrt((hn ** 2).mean()))
        assert np.all(np.abs(acts[l] - hn) <= 1e-4 * np.abs(hn) + 1e-5 * rms), f"{what}: forward of layer {l}"
        flips.append(int(((acts[l] > 0) != (hn > 0)).sum()))
    ratios = {k: _ratio(got[k], want[k]) for k in got}
    chunks, rpc = _plan(N)
    print(f"{what}: N={N} E={E} {chunks} chunks x {rpc} rows, ReLU masks unlike the fp64 forward's per layer {flips}: "
          + ", ".join(f"{k} {r:.3f}" for k, r in ratios.items()))
    for k, r in ratios.items():
        assert r <= 1.0, f"{what} {k}: error ratio {r:.3f}"


@gpu
def test_two_layer_model_on_a_hub_destination_graph():
    """2 layers, F_in = 32, node and edge losses on a 250 003-node hub="dst" graph (2.5 M edges; the largest rows take
    the forward's hub-row path)."""
    N, E = 250_003, 2_500_000
    g = G.synthetic_graph(N=N, E=E, seed=31, hub="dst", f_in=32)
    assert np.diff(g.rowptr.astype(np.int64)).max() > 10_000
    model = GraphSAGE_T(32, HB, 2, seed=31).cuda()
    tg = _train_graph(g.rowptr, g.col, g.ew, False)
    _check_model(model, torch.from_numpy(g.x).cuda(), tg, g.rowptr, g.col, g.ew, 31, "hub dst")


@gpu
def test_two_layer_model_on_a_device_built_stream_window():
    """A window of stream.fleet_columns(1500, 10, seed=0, bystanders=2) built by train.stream_examples (seed 0): 116 130
    nodes, 238 602 edges, largest in-degree and out-degree 3000 each."""
    from nerrf_b200 import stream
    from nerrf_b200.ai import train as T
    cols, _ = stream.fleet_columns(1500, 10, seed=0, bystanders=2)
    ex = T.stream_examples(cols, 1, seed=0, files_per_window=8)[0]
    rowptr, col, ew = ex["rowptr"].cpu().numpy(), ex["col"].cpu().numpy(), ex["ew"].cpu().numpy()
    N = rowptr.size - 1
    rp = rowptr.astype(np.int64)
    print(f"window {ex['window']}: N={N} E={col.size} max in-degree {np.diff(rp).max()} "
          f"max out-degree {np.bincount(col, minlength=N).max()}")
    assert N >= 100_000
    model = GraphSAGE_T(ex["x"].shape[1], HB, 2, seed=7).cuda()
    tg = AG.TrainGraph(ex["rowptr"], ex["col"], ex["ew"])
    _check_model(model, ex["x"], tg, rowptr, col, ew, 7, "stream window")


# -------------------------------------------------------------------------------------------- (c) reproducibility
def _gather_row_weights(rowptr, ew):
    """a_e in fp32 exactly as one warp of gather_row forms it: lane l sums edges e0 + l, e0 + l + 32, ... in order, the
    32 lane sums are combined by the xor butterfly of warp_sum, a_e = w_e * (1 / max(sum, 1e-12))."""
    rp = rowptr.astype(np.int64)
    n, deg = rp.size - 1, np.diff(rp)
    lanes = np.zeros((n, 32), np.float32)
    for k in range(int(-(-deg.max() // 32)) if n else 0):
        for l in range(32):
            j = 32 * k + l
            rows = np.nonzero(deg > j)[0]
            lanes[rows, l] += ew[rp[rows] + j]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    inv = np.float32(1) / np.maximum(lanes[:, 0], np.float32(1e-12))
    return ew * np.repeat(inv, deg)


@gpu
def test_normalised_weights_are_the_forward_aggregates_to_the_bit():
    for rowptr, col, ew in [_graph(3001, 40_000, "dst", seed=2), B.degenerate_graph(500, 4000, 3)]:
        for rp64 in (False, True):
            tg = _train_graph(rowptr, col, ew, rp64)
            order = tg.t_eid.long().cpu().numpy()
            want = _gather_row_weights(rowptr, ew)[order]
            assert np.array_equal(tg.t_w.cpu().numpy().view(np.uint32), want.view(np.uint32))


@gpu
def test_two_constructions_of_a_hub_graph_give_the_same_bits():
    """TrainGraph twice from one hub-destination graph: the same transposed graph bit for bit, and a full forward and
    backward (node and edge losses, x requiring grad) on each gives the same gradient bits."""
    N, E = 100_003, 1_500_000
    g = G.synthetic_graph(N=N, E=E, seed=41, hub="dst", f_in=32)
    tgs = [_train_graph(g.rowptr, g.col, g.ew, False) for _ in range(2)]
    for k in ("t_rowptr", "t_col", "t_w", "t_eid"):
        a, b = getattr(tgs[0], k), getattr(tgs[1], k)
        assert a.dtype == b.dtype and torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                                  b.view(torch.int32) if b.dtype == torch.float32 else b), k
    model = GraphSAGE_T(32, HB, 2, seed=41).cuda()
    rng = np.random.default_rng(41)
    dlogit = torch.from_numpy(rng.standard_normal(N).astype(np.float32)).cuda()
    dedge = torch.from_numpy(rng.standard_normal((E, 2)).astype(np.float32)).cuda()
    runs = []
    for tg in tgs:
        model.zero_grad()
        x = torch.from_numpy(g.x).cuda().requires_grad_()
        nl, el = AG.sage_logits(model, x, tg)
        ((nl * dlogit).sum() + (el * dedge).sum()).backward()
        runs.append([x.grad.clone()] + [p.grad.clone() for p in model.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def test_backward_workspace_is_a_function_of_n_and_F_only(lib_built):
    """The workspace (and with it the chunking of the dW reduction) follows from n and F alone, with the fixed cap of
    264 chunks: a plan that read the device's SM count would differ on a card with another SM count."""
    lib = L.lib()
    need = C.c_size_t()
    for n in (0, 1, 31, 32, 33, 8447, 8448, 8449, 8481, 16_896, 16_897, 100_003, 300_007, 843_000, 10_000_019):
        for F in (32, 64, 128):
            assert lib.nerrf_sage_layer_bwd_workspace_bytes(n, F, C.byref(need)) == 0
            assert need.value == _workspace_bytes(n, F), (n, F)
    assert _plan(8448) == (264, 32) and _plan(8449) == (133, 64) and _plan(100_003) == (261, 384)
    assert _plan(300_007) == (261, 1152)


# ----------------------------------------------------------------------------------- (d) training on an edgeless graph
@gpu
def test_two_layer_model_trains_on_a_graph_without_edges():
    """N > 0, E = 0, x requiring grad: the transposed graph is empty (null t_col / t_w) and dh = dZ[:, :F]."""
    N = 1000
    rowptr, col, ew = B.degenerate_graph(N, 0)
    tg = _train_graph(rowptr, col, ew, False)
    assert tg.t_col.data_ptr() == 0 and tg.t_w.data_ptr() == 0
    model = GraphSAGE_T(32, HB, 2, seed=3).cuda()
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((N, 32)).astype(np.float32)).cuda()
    _check_model(model, x, tg, rowptr, col, ew, 3, "no edges")
