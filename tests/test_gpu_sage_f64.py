"""Every GraphSAGE-T forward kernel against float64 (needs an H100 except the generator test).

The reference is the float64 sparse forward of oracle/sage_bwd_ref.py (pinned against oracle/sage_ref.py by
tests/test_oracle_sage_bwd.py).  The layers are called through nerrf_sage_layer_fwd_ex, whose arguments fix the
instantiation: algo 2 / 3 / 1 = umma (NS = 3) / umma2 (NS = 2) / ffma; the rowptr width; and the hub-row scratch, which
selects UmmaCfg<F, NS, LONG = scratch of at least 8192 bytes>, with RESIDENT = F == 32 || (F == 128 && !LONG).  None
of these tests goes through GraphSAGE_T.forward / layer_forward, whose hub-row answer is cached per rowptr address.

Bounds: the spec's |got - want| <= 1e-4 |want| + atol rms(want), atol = 1e-5 (1e-4 for umma2, tests/gpu_util.py).  The
worst ratio to that bound is printed per case.  On top of it, every umma and ffma output must be within FP32_FACTOR of
the error a plain fp32 evaluation of the same layer (oracle/sage_ref.layer, fp32) makes, in max |error| / rms(want);
umma2 must fail that bound on the same inputs, so the check can tell the 3-term split from the 2-term one."""
import ctypes as C
import functools

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from gpu_util import ATOL_RMS
from nerrf_b200 import _lib as L, graph as G
from nerrf_b200.ai.models import GraphSAGE_T
from oracle import sage_bwd_ref as B, sage_ref as S

gpu = pytest.mark.gpu
H = 128
TN, EMAX, LONG_T, LONG_CH = 32, 512, 128, 256      # sage_umma.cu: tile rows, staged edges, hub-row threshold, chunk
ALGO = {"ffma": 1, "umma": 2, "umma2": 3}
RTOL = 1e-4
# max |got - want| / rms(want) of umma and ffma over that of the fp32 CPU evaluation: at most this factor.  Measured on
# an H100 SXM (700 W) on the boundary graph (DESIGN.md 2.1): umma 2.27x / 2.14x / 3.38x at F = 32 / 64 / 128, ffma
# 1.15x / 0.92x / 1.11x, umma2 15.4x / 8.4x / 7.2x.  umma's margin over fp32 is not the split (leaving
# out x2.w0, one of the products NS = 3 adds to NS = 2's, breaks the spec bound itself) but most likely the wgmma
# accumulation (DESIGN.md 2.1).
FP32_FACTOR = 5.0


# ------------------------------------------------------------------------------------------ the boundary graph
# One 32-row tile per entry: (in-degree, weight kind) per row, the remaining rows of the tile without edges.  Weight
# kinds: "u" 0.5 + 0.5 U(0,1), "tiny" 1e-14 (a row sum below 1e-12), "tiny3" 3e-15 (a hub row summing below 1e-12),
# "zero" 0; "self" self-loops, "multi" one source repeated.
HEAVY_TILES = {
    "511": [(255, "u"), (253, "u"), (3, "u")],                                 # rows from staged offsets 0, 255, 508
    "512": [(512, "u")],                                                        # one 512-edge row from offset 0
    "513": [(256, "u"), (253, "u"), (1, "u"), (1, "u"), (1, "u"), (1, "u")],   # rows from offsets 509, 510, 511, 512
    "513b": [(385, "u"), (128, "u")],                                           # a 128-edge row across the staged end
    "2k": [(130, "u"), (383, "u"), (384, "u"), (257, "u"), (513, "u"), (129, "u"), (127, "u"), (1, "u"), (0, "u")]
          + [(24, "u")] * 22,                                                   # 2452 edges, rows far past offset 512
    "4097": [(4097, "u")] + [(3, "u")] * 31,
    "degenerate": [(6, "tiny"), (4, "zero"), (5, "self"), (7, "multi"), (0, "u"), (300, "tiny3"), (300, "zero"),
                   (3, "u"), (2, "self"), (9, "multi")],
}
HUGE_TILE = [(65_537, "u"), (2, "u"), (0, "u"), (1, "u")]
REQUIRED_DEGREES = (0, 1, 127, 128, 129, 130, 255, 256, 257, 383, 384, 385, 512, 513, 4097)


@functools.lru_cache(maxsize=None)
def boundary_graph(seed=7):
    """-> (rowptr int32, col int32, ew float32) of 40 019 nodes: light tiles (0-20 in-edges per row, ~320 per tile)
    around two runs of the HEAVY_TILES kinds, the second run shifted by an odd number of tiles (each kind at an even and
    an odd tile index; which slot of a tile pair a tile lands in is decided by the dynamic tile schedule), a third run
    after the 65 537-edge row, and a partial last tile of 19 rows."""
    rng = np.random.default_rng(seed)
    light = lambda: [(int(d), "u") for d in rng.integers(0, 21, TN)]
    kinds = list(HEAVY_TILES.values())
    tiles = [light() for _ in range(40)] + kinds + [light(), light()] + kinds + [light() for _ in range(300)]
    tiles += [HUGE_TILE] + [light() for _ in range(200)] + kinds
    n_tiles = 1250
    tiles += [light() for _ in range(n_tiles - len(tiles))]
    N = n_tiles * TN + 19
    rows = [r for t in tiles for r in (t + [(0, "u")] * (TN - len(t)))][:N]
    rows += [(int(d), "u") for d in rng.integers(0, 21, N - len(rows))]
    deg = np.array([d for d, _ in rows], np.int64)
    rowptr = np.zeros(N + 1, np.int64)
    np.cumsum(deg, out=rowptr[1:])
    col = rng.integers(0, N, int(rowptr[-1])).astype(np.int32)
    ew = (0.5 + 0.5 * rng.random(col.size)).astype(np.float32)
    for v, (d, kind) in enumerate(rows):
        e0, e1 = rowptr[v], rowptr[v + 1]
        if kind in ("tiny", "tiny3", "zero"):
            ew[e0:e1] = {"tiny": 1e-14, "tiny3": 3e-15, "zero": 0.0}[kind]
        elif kind == "self":
            col[e0:e1] = v
        elif kind == "multi":
            col[e0:e1 - 2] = col[e0]
    assert rowptr[-1] < 2 ** 31
    return rowptr.astype(np.int32), col, ew


def test_boundary_graph_has_its_boundaries():
    """The generator's CSR has every boundary the GPU tests rely on (a change to it cannot silently drop one)."""
    rowptr, col, ew = boundary_graph()
    rp = rowptr.astype(np.int64)
    N = rp.size - 1
    deg = np.diff(rp)
    assert 30_000 <= N <= 60_000 and N % TN != 0                                   # a partial last tile
    n_tiles = -(-N // TN)
    t0 = rp[np.minimum(np.arange(n_tiles) * TN, N)]
    tile_e = rp[np.minimum(np.arange(1, n_tiles + 1) * TN, N)] - t0
    for want in (511, 512, 513):
        at = np.flatnonzero(tile_e == want)
        assert {0, 1} <= set(at % 2), f"a {want}-edge tile at an even and an odd tile index"
    at = np.flatnonzero(tile_e > 2000)
    assert {0, 1} <= set(at % 2)
    assert (tile_e[at[:-1] + 1] > EMAX).any() and (tile_e[at[:-1] + 1] <= EMAX).any()   # heavy and light neighbours
    assert 256 <= np.median(tile_e) <= 384
    off = rp[:-1] - t0[np.arange(N) // TN]                                         # staged offset of each row's first edge
    starts = set(off[deg > 0].tolist())
    assert {0, 508, 509, 510, 511, 512} <= starts and max(starts) > EMAX
    assert ((deg == 512) & (off == 0)).any()
    assert ((off < EMAX) & (off + deg > EMAX)).any()                               # rows across the staged end
    assert set(REQUIRED_DEGREES) <= set(deg.tolist()) and deg.max() >= 65_537
    # degenerate rows (oracle/sage_bwd_ref.degenerate_graph's kinds, plus two hub rows)
    dst = B.edge_dst(rp)
    wsum = np.bincount(dst, weights=ew.astype(np.float64), minlength=N)
    assert ((deg > 0) & (deg <= LONG_T) & (wsum > 0) & (wsum < 1e-12)).any()
    assert ((deg > 0) & (deg <= LONG_T) & (wsum == 0)).any()
    assert ((deg > LONG_T) & (wsum > 0) & (wsum < 1e-12)).any()
    assert ((deg > LONG_T) & (wsum == 0)).any()
    assert (col == dst).any()                                                       # self-loops
    pairs = dst * N + col
    assert np.unique(pairs).size < pairs.size                                       # multi-edges
    assert (deg == 0).sum() > 100


# ------------------------------------------------------------------------------------------ helpers
def long_ws_capacity(nbytes):
    """Chunk items a hub-row scratch of `nbytes` holds (sage_umma.cu long_ws_carve)."""
    if nbytes < 8192:
        return 0
    cap = ((nbytes - 256) // (8 + 128 * 4 + 4 + 32)) & ~3
    slots = 1 << (2 * cap - 1).bit_length()
    while 256 + slots * 8 + cap * (8 + 128 * 4 + 4) > nbytes and cap > 4:
        cap = (cap * 3 // 4) & ~3
        slots = 1 << (2 * cap - 1).bit_length()
    return cap


def chunk_items(deg):
    """Chunk items the hub rows of a graph take in the scratch."""
    deg = np.asarray(deg, np.int64)
    return int((-(-deg[deg > LONG_T] // LONG_CH)).sum())


def scratch(mode, deg, n_edges):
    """The hub-row scratch of a mode: None ("none", LONG off), the library's size for the graph ("full"), or a third of
    the chunk items the graph's hub rows need ("mix": the rows that fit are pre-aggregated, the rest stay inline)."""
    if mode == "none":
        return None
    if mode == "full":
        need = C.c_size_t()
        L.check(L.lib().nerrf_sage_long_rows_workspace_bytes(int(n_edges), C.byref(need)), "long_rows_workspace_bytes")
        nbytes = need.value
        assert long_ws_capacity(nbytes) >= chunk_items(deg)
    else:
        items = chunk_items(deg)
        nbytes = 256 + (items // 3) * 580
        assert 0 < long_ws_capacity(nbytes) < items
    return torch.empty(nbytes, dtype=torch.uint8, device="cuda")


def fwd(x, rp, colp, ewp, W, b, out, rb, re, algo, ws=None, relu=True, node_w=None, node_b=0.0, score=None):
    """One nerrf_sage_layer_fwd_ex call: the arguments alone pick the instantiation."""
    N, F = x.shape
    L.check(L.lib().nerrf_sage_layer_fwd_ex(
        L.ptr(x), L.ptr(rp), int(rp.dtype == torch.int64), colp, ewp, L.ptr(W), L.ptr(b), L.ptr(out), N, rb, re, F, H,
        int(relu), ALGO[algo], L.ptr(node_w), float(node_b), L.ptr(score), L.ptr(ws), 0 if ws is None else ws.numel(),
        None, 0, None, L.current_stream_ptr()), "nerrf_sage_layer_fwd_ex")


def ratio(got, want, atol=1e-5):
    """max |got - want| / (RTOL |want| + atol rms(want)): <= 1 is inside the spec bound."""
    got = np.asarray(got.detach().cpu().numpy() if hasattr(got, "detach") else got, np.float64)
    want = np.asarray(want, np.float64)
    assert got.shape == want.shape
    if want.size == 0:
        return 0.0
    rms = max(float(np.sqrt((want ** 2).mean())), 1e-30)
    return float((np.abs(got - want) / (RTOL * np.abs(want) + atol * rms)).max())


def rel_err(got, want):
    """max |got - want| / rms(want)"""
    got = np.asarray(got.detach().cpu().numpy() if hasattr(got, "detach") else got, np.float64)
    want = np.asarray(want, np.float64)
    return float(np.abs(got - want).max() / max(float(np.sqrt((want ** 2).mean())), 1e-30))


def sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------------------------------ (b-d) the matrix
@gpu
@pytest.mark.parametrize("F", [32, 64, 128])
def test_layer_instantiations_against_float64_on_the_boundary_graph(F):
    """Each of umma, umma2 and ffma; int32 and int64 rowptr; hub-row scratch none / full / mix (umma, umma2); ReLU on and
    off; fused node head on and off; rows [0, N) and [13, N - 7).  Against the float64 layer (one evaluation per F):
    every output within the spec bound, umma and ffma within FP32_FACTOR of the fp32 evaluation's error, umma2 outside
    it.  Bit equalities: int32 = int64 rowptr, a range = the same rows of the full call, head on = head off, a second
    launch = the first, and rows with at most 128 in-edges equal between LONG on and off."""
    rowptr, col, ew = boundary_graph()
    N = rowptr.size - 1
    deg = np.diff(rowptr.astype(np.int64))
    rng = np.random.default_rng(F)
    xn = rng.standard_normal((N, F)).astype(np.float32)
    model = GraphSAGE_T(F, H, 1, seed=F)
    Wn, bn = model.weights[0].detach().numpy(), model.biases[0].detach().numpy()
    nwn, nb = model.node_w.detach().numpy(), float(model.node_b.detach()[0])
    z64, _ = B.layer_forward(xn, rowptr, col, ew, Wn, bn, relu=False, sparse=True)
    z32 = S.layer(torch.from_numpy(xn), torch.from_numpy(rowptr), torch.from_numpy(col), torch.from_numpy(ew),
                  torch.from_numpy(Wn), torch.from_numpy(bn), relu=False).numpy()
    x, W, b, nw = dev(xn), dev(Wn), dev(bn), dev(nwn)
    rps = {False: dev(rowptr), True: dev(rowptr.astype(np.int64))}
    dcol, dew = dev(col), dev(ew)
    colp, ewp = L.ptr(dcol), L.ptr(dew)
    ranges = {"full": (0, N), "off-grid": (13, N - 7)}
    ref = {(relu, rn): np.maximum(z64[rb:re], 0) if relu else z64[rb:re]
           for relu in (1, 0) for rn, (rb, re) in ranges.items()}
    e32 = {(relu, rn): rel_err(np.maximum(z32[rb:re], 0) if relu else z32[rb:re], ref[(relu, rn)])
           for relu in (1, 0) for rn, (rb, re) in ranges.items()}
    small = torch.from_numpy(deg <= LONG_T).cuda()
    worst_factor = {}
    print(f"\nF={F} N={N} E={col.size}: fp32 evaluation max|err|/rms = {max(e32.values()):.2e}")
    for algo in ("umma", "umma2", "ffma"):
        atol = ATOL_RMS[algo]
        plain = {}
        for mode in (("none", "full", "mix") if algo != "ffma" else ("none",)):
            ws = scratch(mode, deg, col.size)
            outs = {}
            for rp64 in (False, True):
                worst, fac = 0.0, 0.0
                for relu in (1, 0):
                    for head in (False, True):
                        for rn, (rb, re) in ranges.items():
                            out = torch.full((N, H), -7.0, device="cuda")
                            score = torch.full((N,), -7.0, device="cuda") if head else None
                            fwd(x, rps[rp64], colp, ewp, W, b, out, rb, re, algo, ws, relu,
                                nw if head else None, nb, score)
                            torch.cuda.synchronize()
                            what = f"F={F} {algo} rp{64 if rp64 else 32} {mode} relu={relu} head={head} {rn}"
                            assert bool((out[:rb] == -7).all()) and bool((out[re:] == -7).all()), what
                            r = ratio(out[rb:re], ref[(relu, rn)], atol)
                            assert r <= 1.0, f"{what}: error ratio {r:.3f}"
                            worst = max(worst, r)
                            fac = max(fac, rel_err(out[rb:re], ref[(relu, rn)]) / e32[(relu, rn)])
                            if head:
                                h64 = out[rb:re].double().cpu().numpy()
                                rs = ratio(score[rb:re], sigmoid(h64 @ nwn.astype(np.float64) + nb))
                                assert rs <= 1.0, f"{what}: node score error ratio {rs:.3f}"
                                assert bool((score[:rb] == -7).all()) and bool((score[re:] == -7).all()), what
                            outs[(rp64, relu, head, rn)] = out
                worst_factor[(algo, mode, rp64)] = fac
                print(f"  {algo:5s} rp{64 if rp64 else 32} scratch {mode:4s}: worst spec ratio {worst:.3f}, "
                      f"max|err|/rms {fac:.2f}x the fp32 evaluation's")
            if mode != "mix":           # which hub rows fit a too-small scratch depends on the scan's atomics: no bit claims
                for key, out in outs.items():
                    rp64, relu, head, rn = key
                    rb, re = ranges[rn]
                    assert torch.equal(out, outs[(not rp64, relu, head, rn)]), f"{algo} {mode} int32 vs int64 {key}"
                    assert torch.equal(out[rb:re], outs[(rp64, relu, head, "full")][rb:re]), f"{algo} {mode} range {key}"
                    assert torch.equal(out, outs[(rp64, relu, not head, rn)]), f"{algo} {mode} head on / off {key}"
                again = torch.empty(N, H, device="cuda")
                fwd(x, rps[False], colp, ewp, W, b, again, 0, N, algo, ws, 1)
                torch.cuda.synchronize()
                assert torch.equal(again, outs[(False, 1, False, "full")]), f"{algo} {mode}: second launch"
            plain[mode] = outs[(False, 1, False, "full")]
        for mode in plain:
            assert torch.equal(plain[mode][small], plain["none"][small]), f"{algo}: rows <= 128 in-edges, LONG {mode}"
    umma_f = max(v for (a, _, _), v in worst_factor.items() if a != "umma2")
    umma2_f = min(v for (a, _, _), v in worst_factor.items() if a == "umma2")
    assert umma_f <= FP32_FACTOR, f"umma / ffma error {umma_f:.2f}x the fp32 evaluation's"
    assert umma2_f > FP32_FACTOR, f"umma2 error only {umma2_f:.2f}x the fp32 evaluation's: the check is too weak"


# ------------------------------------------------------------------------------------------ (e) the small entry points
@gpu
def test_aggregate_and_heads_against_float64_on_the_boundary_graph():
    """nerrf_sage_aggregate (F = 32, 64, 128), nerrf_sage_node_head (score and proj) and nerrf_sage_edge_head with int32
    and int64 rowptr: the same bits for both widths, within the spec bound of float64 evaluated at the device's inputs."""
    rowptr, col, ew = boundary_graph()
    N = rowptr.size - 1
    deg = np.diff(rowptr.astype(np.int64))
    rps = {False: dev(rowptr), True: dev(rowptr.astype(np.int64))}
    dcol, dew = dev(col), dev(ew)
    rng = np.random.default_rng(3)
    for F in (32, 64, 128):
        xn = rng.standard_normal((N, F)).astype(np.float32)
        x = dev(xn)
        want = B.aggregate(xn, rowptr, col, ew, sparse=True)
        ms = []
        for rp64 in (False, True):
            m = torch.full((N, F), -7.0, device="cuda")
            L.check(L.lib().nerrf_sage_aggregate(L.ptr(x), L.ptr(rps[rp64]), int(rp64), L.ptr(dcol), L.ptr(dew), L.ptr(m),
                                                 N, 0, N, F, L.current_stream_ptr()), "nerrf_sage_aggregate")
            ms.append(m)
        torch.cuda.synchronize()
        r = ratio(ms[0], want)
        print(f"aggregate F={F}: spec ratio {r:.3f}")
        assert r <= 1.0 and torch.equal(ms[0], ms[1])
        assert bool((ms[0][torch.from_numpy(deg == 0).cuda()] == 0).all())
    model = GraphSAGE_T(128, H, 1, seed=5)
    hn = np.maximum(rng.standard_normal((N, H)), 0).astype(np.float32)
    h = dev(hn)
    nw, eW, eb = (p.detach().cuda() for p in (model.node_w, model.edge_W, model.edge_b))
    nb = float(model.node_b.detach()[0])
    score = torch.empty(N, device="cuda")
    proj = torch.empty(N, 4, device="cuda")
    L.check(L.lib().nerrf_sage_node_head(L.ptr(h), L.ptr(nw), nb, L.ptr(score), L.ptr(eW), L.ptr(proj), 0, N, H,
                                         L.current_stream_ptr()), "nerrf_sage_node_head")
    h64, eW64 = hn.astype(np.float64), eW.double().cpu().numpy()
    want_p = np.concatenate([h64 @ eW64[:H], h64 @ eW64[H:]], 1)
    rs = ratio(score, sigmoid(h64 @ nw.double().cpu().numpy() + nb))
    rp_ = ratio(proj, want_p)
    print(f"node head: score {rs:.3f}, proj {rp_:.3f}")
    assert rs <= 1.0 and rp_ <= 1.0
    logits = []
    for rp64 in (False, True):
        el = torch.empty(col.size, 2, device="cuda")
        L.check(L.lib().nerrf_sage_edge_head(L.ptr(proj), L.ptr(rps[rp64]), int(rp64), L.ptr(dcol), L.ptr(eb), L.ptr(el),
                                             0, N, L.current_stream_ptr()), "nerrf_sage_edge_head")
        logits.append(el)
    torch.cuda.synchronize()
    p = proj.double().cpu().numpy()
    dst = B.edge_dst(rowptr)
    want_e = p[col][:, :2] + p[dst][:, 2:] + eb.double().cpu().numpy()
    re_ = ratio(logits[0], want_e)
    print(f"edge head: {re_:.3f}")
    assert re_ <= 1.0 and torch.equal(logits[0], logits[1])


# ------------------------------------------------------------------------------------------ (f) bench scale
def _bench_graph(family):
    """-> (rowptr, col, ew, x) of the cfg-2 families of test_gpu_sage.test_full_size_forward_vs_oracle, the F = 64
    hub-destination graph, or a device-built fleet window."""
    if family == "uniform":
        rng = np.random.Generator(np.random.PCG64(77))
        N, E = 1_000_000, 10_000_000
        rowptr, col, ew = G.csr_from_edges(rng.integers(0, N, E), rng.integers(0, N, E),
                                           (rng.random(E) * 60).astype(np.float32),
                                           (0.5 + 0.5 * rng.random(E)).astype(np.float32), N)
        return rowptr, col, ew, np.random.Generator(np.random.PCG64(0)).standard_normal((N, 32), dtype=np.float32)
    if family == "window":
        from nerrf_b200 import stream
        from nerrf_b200.ai import train as T
        cols, _ = stream.fleet_columns(1500, 10, seed=0, bystanders=2)
        ex = T.stream_examples(cols, 1, seed=0, files_per_window=8)[0]
        return (ex["rowptr"].cpu().numpy(), ex["col"].cpu().numpy(), ex["ew"].cpu().numpy(),
                np.ascontiguousarray(ex["x"].cpu().numpy()))
    g = G.synthetic_graph(hub="dst" if "dst" in family else "src", f_in=64 if family.startswith("f64") else 32)
    return g.rowptr, g.col, g.ew, g.x


@gpu
@pytest.mark.parametrize("family", ["hub_src", "hub_dst", "uniform", "f64_hub_dst", "window"])
def test_bench_scale_forward_layer_by_layer_against_float64(family):
    """Three umma layers with the hub-row scratch when the graph has hub rows (as the model picks it): each layer within
    the spec bound of float64 evaluated at the device's previous layer output (ReLU masks flip across layers), with the
    C oracle's own distance printed beside it; nerrf_sage_forward gives the same bits, and its h, node scores and top-64
    ranking match the C oracle's whole forward under test_gpu_sage's rules."""
    from oracle import c_sage
    from test_gpu_sage import _ranking_matches
    from gpu_util import assert_close_fp32
    rowptr, col, ew, xn = _bench_graph(family)
    N, F = xn.shape
    deg = np.diff(rowptr.astype(np.int64))
    hub = bool(deg.max() > LONG_T)
    model = GraphSAGE_T(F, H, 3, seed=1)
    P = model.oracle_params()
    rp, dcol, dew = dev(rowptr), dev(col), dev(ew)
    ws = scratch("full", deg, col.size) if hub else None
    print(f"\n{family}: N={N} E={col.size} F={F} max in-degree {deg.max()}, hub-row scratch {'on' if hub else 'off'}")
    h = dev(xn)
    for l, (Wc, bc) in enumerate(P["layers"]):
        W, b = dev(Wc.numpy()), dev(bc.numpy())
        out = torch.empty(N, H, device="cuda")
        fwd(h, rp, L.ptr(dcol), L.ptr(dew), W, b, out, 0, N, "umma", ws)
        torch.cuda.synchronize()
        hp = h.cpu().numpy()
        want, _ = B.layer_forward(hp, rowptr, col, ew, Wc.numpy(), bc.numpy(), sparse=True)
        rk = ratio(out, want)
        rc = ratio(c_sage.layer(hp, rowptr, col, ew, Wc.numpy(), bc.numpy()), want)
        print(f"  layer {l}: kernel spec ratio {rk:.3f}, C oracle {rc:.3f}; max|err|/rms kernel "
              f"{rel_err(out, want):.2e}")
        assert rk <= 1.0, f"{family} layer {l}: error ratio {rk:.3f}"
        h = out
    pp = ((N * H * 4 + 255) // 256) * 256
    wsf = torch.empty(pp + (ws.numel() if hub else 0), dtype=torch.uint8, device="cuda")
    hf, sc = torch.empty(N, H, device="cuda"), torch.empty(N, device="cuda")
    Ws = [dev(w.numpy()) for w, _ in P["layers"]]
    bs = [dev(b_.numpy()) for _, b_ in P["layers"]]
    nw = dev(P["node_w"].numpy())
    L.check(L.lib().nerrf_sage_forward(L.ptr(dev(xn)), L.ptr(rp), int(rp.dtype == torch.int64), L.ptr(dcol), L.ptr(dew),
                                       N, F, H, 3, L.ptr_array(Ws), L.ptr_array(bs), L.ptr(nw),
                                       float(P["node_b"][0]), L.ptr(hf), L.ptr(sc), L.ptr(wsf), wsf.numel(), ALGO["umma"],
                                       L.current_stream_ptr()), "nerrf_sage_forward")
    torch.cuda.synchronize()
    assert torch.equal(hf, h), "nerrf_sage_forward vs the layer calls"
    hw, scw = c_sage.forward(P, xn, rowptr, col, ew)
    assert_close_fp32(hf, torch.from_numpy(hw), what=f"{family} h")
    err = float(np.abs(sc.cpu().numpy() - scw).max())
    assert err < 1e-5, f"node scores differ by {err}"
    safe = _ranking_matches(sc.cpu().numpy(), scw, 64, err)
    print(f"  whole forward: score max err {err:.2e}, top-64 exact for the first {safe} ranks")


# ------------------------------------------------------------------------------------------ (g) past 2^31 edges
DEG_BLOCK = (0, 1, 100, 129, 513, 900, 1000, 1461)      # 4104 = 8 x 513 edges per 8 rows


@gpu
def test_int64_rowptr_past_2_31_edges():
    """2^22 nodes, 2^31 + 2^22 edges (in-degrees DEG_BLOCK repeated; the row holding edge 2^31 is a 1461-edge hub row),
    sources uniform.  F = 32 and 128: umma with no scratch and with a full one, and ffma (which has no hub-row path);
    ~2000 sampled rows (the straddling row and its neighbours, the last row, rows on both sides of 2^31) against float64
    from their own slices, and every row bit for bit against two int32-rowptr windows over the same arrays (rowptr
    minus the window's first edge, col / ew pointers advanced by it).  nerrf_sage_aggregate likewise."""
    N = 1 << 22
    E = N * 513
    block = torch.tensor(DEG_BLOCK, dtype=torch.int64)
    assert int(block.sum()) == 8 * 513
    items = chunk_items(np.array(DEG_BLOCK)) * (N // 8)
    ws_bytes = 256 + items * 580 + 4096
    assert long_ws_capacity(ws_bytes) >= items
    need = 8 * E + 8 * N + 8 * N + 3 * N * H * 4 + ws_bytes + (2 << 30)
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")
    try:
        _past_2_31(N, E, block, ws_bytes)
    finally:
        torch.cuda.empty_cache()


def _past_2_31(N, E, block, ws_bytes):
    rp = torch.zeros(N + 1, dtype=torch.int64, device="cuda")
    rp[1:] = torch.cumsum(block.cuda().repeat(N // 8), 0)
    assert int(rp[-1]) == E
    col = torch.empty(E, dtype=torch.int32, device="cuda")
    ew = torch.empty(E, dtype=torch.float32, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(31)
    CH = 1 << 28                                                        # 1 GB per chunk, no larger temporary
    for a in range(0, E, CH):
        col[a:a + CH].random_(0, N, generator=gen)
        ew[a:a + CH].uniform_(0.5, 1.0, generator=gen)
    rph = rp.cpu().numpy()
    straddle = int(np.searchsorted(rph, 2 ** 31, side="right")) - 1
    assert rph[straddle] < 2 ** 31 < rph[straddle + 1] and rph[straddle + 1] - rph[straddle] > LONG_T
    # windows: rows [0, r1) with base 0 and rows [r1, N) with base rowptr[r1]; each below 2^31 edges
    r1 = N // 2
    base = int(rph[r1])
    assert base < 2 ** 31 and E - base < 2 ** 31 and rph[r1] <= rph[straddle]
    rp_a = rp.clamp(max=base).to(torch.int32)
    rp_b = (rp.clamp(min=base) - base).to(torch.int32)
    windows = [(rp_a, 0, 0, r1), (rp_b, base, r1, N)]
    # sampled rows and their slices
    rng = np.random.default_rng(31)
    above = np.flatnonzero(rph[:-1] >= 2 ** 31)
    sample = np.unique(np.concatenate([[straddle - 1, straddle, straddle + 1, N - 1, 0], rng.choice(above, 700),
                                       rng.choice(np.flatnonzero(rph[:-1] < 2 ** 31), 700), rng.integers(0, N, 600)]))
    deg = np.diff(rph)[sample]
    eidx = torch.from_numpy(np.concatenate([np.arange(rph[v], rph[v + 1]) for v in sample])).cuda()
    s_col, s_ew = col[eidx].cpu().numpy(), ew[eidx].cpu().numpy().astype(np.float64)
    s_rp = np.concatenate([[0], np.cumsum(deg)])
    wsum = np.bincount(np.repeat(np.arange(sample.size), deg), weights=s_ew, minlength=sample.size)
    print(f"\nE={E} N={N}: row {straddle} holds edge 2^31 ({rph[straddle]}..{rph[straddle + 1]}); "
          f"{sample.size} sampled rows, {(rph[sample] >= 2 ** 31).sum()} of them past 2^31")
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    out = torch.empty(N, H, device="cuda")
    out_w = torch.empty(N, H, device="cuda")
    for F in (32, 128):
        x = torch.empty(N, F, device="cuda").normal_(generator=gen)
        need_rows = np.unique(np.concatenate([sample, s_col]))
        xs = x[torch.from_numpy(need_rows).cuda()].double().cpu().numpy()
        pos = lambda ids: np.searchsorted(need_rows, ids)
        A = sp.csr_matrix((s_ew / np.maximum(np.repeat(wsum, deg), 1e-12), pos(s_col), s_rp),
                          shape=(sample.size, need_rows.size))
        m64 = np.asarray(A @ xs)
        model = GraphSAGE_T(F, H, 1, seed=F)
        Wn, bn = model.weights[0].detach().double().numpy(), model.biases[0].detach().double().numpy()
        W, b = model.weights[0].detach().cuda(), model.biases[0].detach().cuda()
        want = np.maximum(np.concatenate([xs[pos(sample)], m64], 1) @ Wn + bn, 0)
        for algo, ws_ in (("umma", None), ("umma", ws), ("ffma", None)):
            what = f"F={F} {algo} scratch {'on' if ws_ is not None else 'off'}"
            fwd(x, rp, L.ptr(col), L.ptr(ew), W, b, out, 0, N, algo, ws_)
            for rpw, eb, rb, re in windows:
                fwd(x, rpw, C.c_void_p(col.data_ptr() + 4 * eb), C.c_void_p(ew.data_ptr() + 4 * eb), W, b, out_w, rb, re,
                    algo, ws_)
            torch.cuda.synchronize()
            r = ratio(out[torch.from_numpy(sample).cuda()], want)
            print(f"  {what}: sampled rows spec ratio {r:.3f}")
            assert r <= 1.0, f"{what}: error ratio {r:.3f}"
            assert torch.equal(out, out_w), f"{what}: int64 rowptr vs int32 windows"
        m = out[:, :F] if F == H else torch.empty(N, F, device="cuda")
        m_w = out_w[:, :F] if F == H else torch.empty(N, F, device="cuda")
        L.check(L.lib().nerrf_sage_aggregate(L.ptr(x), L.ptr(rp), 1, L.ptr(col), L.ptr(ew), L.ptr(m), N, 0, N, F,
                                             L.current_stream_ptr()), "nerrf_sage_aggregate")
        for rpw, eb, rb, re in windows:
            L.check(L.lib().nerrf_sage_aggregate(L.ptr(x), L.ptr(rpw), 0, C.c_void_p(col.data_ptr() + 4 * eb),
                                                 C.c_void_p(ew.data_ptr() + 4 * eb), C.c_void_p(m_w.data_ptr() + 4 * rb * F),
                                                 N, rb, re, F, L.current_stream_ptr()), "nerrf_sage_aggregate")
        torch.cuda.synchronize()
        r = ratio(m[torch.from_numpy(sample).cuda()], m64)
        print(f"  F={F} aggregate: sampled rows spec ratio {r:.3f}")
        assert r <= 1.0 and torch.equal(m, m_w)
        del x
