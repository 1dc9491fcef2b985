"""The 1-D sharded GraphSAGE-T layer path (nerrf_b200.dist) on one GPU: every rank of a sharded forward is emulated
in turn, in layer-major order (the order the per-layer barrier enforces on real ranks), each with its own model.

A rank's layer call addresses its edge block with absolute edge offsets (edge_base), covers only its row range, and in
the fused exchange also stores its rows into the peers' buffers; a peer buffer is just a device pointer, so a
same-device tensor stands in for it.  Everything is checked against (a) the single-GPU forward of the full graph,
bit for bit, and (b) the fp64 oracle."""
import functools

import numpy as np
import pytest
import torch

from nerrf_b200 import _lib as L, dist as D, graph as G
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.ai.models.graphsage_t import ALGOS as ALGO_CODE
from oracle import sage_ref as S
from gpu_util import ATOL_RMS, assert_close_fp32

pytestmark = pytest.mark.gpu

LAYERS = 3
H = 128
LONG_T, LONG_CH = 128, 256            # the kernel's hub-row threshold and chunk length (sage_umma.cu)
N_SYN, E_SYN = 24_000, 360_000        # hub_dst: row 0 has ~12k in-edges, ~240 rows have more than LONG_T
TRACE_COMPONENTS, TRACE_S = 500, 64   # 32k nodes, ~315k edges: every 64th node is a process row with ~300 in-edges
NAN = float("nan")


# ----------------------------------------------------------------------------------------------- graphs and shards
@functools.lru_cache(maxsize=None)
def graph(name, F):
    """(rowptr int32, col, ew, x [N, F]) as host arrays; "trace" is dist.gpu_trace_graph's component structure."""
    if name == "trace":
        rp, col, ew, _, s = D.gpu_trace_graph(TRACE_COMPONENTS, "cuda")
        assert s == TRACE_S
        rp, col, ew = (t.cpu().numpy() for t in (rp, col, ew))
        return rp, col, ew, np.random.default_rng(F).standard_normal((rp.size - 1, F), dtype=np.float32)
    g = G.synthetic_graph(N=N_SYN, E=E_SYN, seed=3, hub=name[4:], f_in=F)
    return g.rowptr, g.col, g.ew, g.x


def family_graph(family):
    """-> (graph name, Shard align) of a test family; trace_aligned cuts only between components."""
    return ("trace", TRACE_S) if family == "trace_aligned" else (family, 1)


def offset_view(t, off=3):
    """A copy of `t` living `off` elements into a larger device buffer (a view whose pointer is not 16-byte aligned)."""
    buf = torch.zeros(t.numel() + 8, dtype=t.dtype, device="cuda")
    v = buf[off:off + t.numel()]
    v.copy_(t)
    return v


def make_shards(rp, col, ew, world, source, cut="edges", align=1, cuts=None, monkeypatch=None):
    """One dist.Shard per rank.  source: "host" (numpy arrays: every rank's edge block is a fresh allocation, as in
    ShardedSage.sharded_upload and bench.py), "device" (the blocks are views into the full device arrays) or "offset"
    (views into device arrays that start 3 elements into a larger buffer).  cuts: explicit row cuts [world + 1]."""
    if source != "host":
        rp, col, ew = (torch.from_numpy(a).cuda() for a in (rp, col, ew))
        if source == "offset":
            col, ew = offset_view(col), offset_view(ew)
            assert col.data_ptr() % 16 and ew.data_ptr() % 16
    if cuts is None:
        return [D.Shard(rp, col, ew, r, world, device="cuda", cut=cut, align=align) for r in range(world)]
    with monkeypatch.context() as mp:
        mp.setattr(G, "edge_balanced_row_cuts", lambda rowptr, parts: np.asarray(cuts, dtype=np.int64))
        shards = [D.Shard(rp, col, ew, r, world, device="cuda") for r in range(world)]
    assert list(shards[0].cuts) == list(cuts)
    return shards


def need_masks(rowptr, col, cuts):
    """uint8 [N] per rank: bit s of rank r's mask is set where the s-th OTHER rank (ascending, skipping r: the slot order
    of PeerBuffers.peers) has the row as a source in its edge block."""
    N, world = rowptr.size - 1, len(cuts) - 1
    reads = []
    for p in range(world):
        m = np.zeros(N, np.uint8)
        m[col[rowptr[cuts[p]]:rowptr[cuts[p + 1]]]] = 1
        reads.append(m)
    masks = []
    for r in range(world):
        mask = np.zeros(N, np.uint8)
        for s, p in enumerate(q for q in range(world) if q != r):
            mask |= reads[p] << s
        masks.append(mask)
    return masks


# ----------------------------------------------------------------------------------------------- references
def make_models(F, algo, n):
    """n models with identical weights (one per emulated rank, each with its own hub-row scratch)."""
    p = GraphSAGE_T(F, H, LAYERS, algo=algo).oracle_params()
    return [GraphSAGE_T(F, H, LAYERS, algo=algo).cuda().load_oracle_params(p) for _ in range(n)]


def single_gpu(model, x, rp, col, ew):
    """(a): the single-GPU forward of the full graph, layer by layer -> ([h_1 .. h_L], scores)."""
    hs, h = [], x
    score = torch.empty(x.shape[0], device="cuda")
    for l in range(LAYERS):
        h = model.layer_forward(l, h, rp, col, ew, score_out=score if l == LAYERS - 1 else None, reuse_long_scan=l > 0)
        hs.append(h)
    return hs, score


def wants_oracle(family, algo, F):
    return family in ("hub_dst", "trace") and (algo == "umma" or F == 32)


def check_oracle(name, F, algo, hs, score, what):
    """(b): every layer of a sharded forward against the fp64 oracle layer applied to that layer's input, and the
    scores against the fp64 node head.  Layer by layer, because the per-layer bound does not hold for three chained
    tensor-core layers at F=128: each umma layer stays within it, but its error (about 3x the fp32 CUDA-core layer's,
    from accumulating six bf16 products per K step on the tensor cores) compounds through the next layers."""
    rp, col, ew, x = graph(name, F)
    p = GraphSAGE_T(F, H, LAYERS).oracle_params()
    t = torch.from_numpy
    dst = S.edge_dst(t(rp))
    h_in = t(x)
    for l, (W, b) in enumerate(p["layers"]):
        want = S.layer(h_in, t(rp), t(col), t(ew), W, b, dst=dst, dtype=torch.float64)
        assert_close_fp32(hs[l], want, atol_rms=ATOL_RMS[algo], what=f"{what}: layer {l} vs fp64 oracle")
        h_in = hs[l].cpu()
    want = torch.sigmoid(h_in.double() @ p["node_w"].double() + p["node_b"].double())
    assert_close_fp32(score, want, atol_rms=ATOL_RMS[algo], what=f"{what}: scores vs fp64 oracle")


def bits(t):
    return t.contiguous().view(torch.int32)


# ----------------------------------------------------------------------------------------------- 1. NCCL-style exchange
def emulate_allgather(models, shards, x, ref, what):
    """Sharded forward with the collective exchange: every rank computes its rows of a layer into its own NaN-filled
    buffer, then its rows are copied into the next layer's shared input (the all-gather).  Checks each rank's rows of
    every layer and its scores against the single-GPU forward, and that nothing outside its rows was written.
    -> ([gathered output of every layer], scores)."""
    ref_h, ref_score = ref
    N = x.shape[0]
    layer = [D.cuda_layer_fn(m) for m in models]
    h, hs = x, []
    score = torch.full((N,), NAN, device="cuda")
    for l in range(LAYERS):
        last = l == LAYERS - 1
        gathered = torch.full((N, H), NAN, device="cuda")
        for r, sh in enumerate(shards):
            rb, re = sh.row_begin, sh.row_end
            out = torch.full((N, H), NAN, device="cuda")
            sc = torch.full((N,), NAN, device="cuda") if last else None
            layer[r](l, h, out, sh, score_out=sc)
            assert torch.equal(out[rb:re], ref_h[l][rb:re]), f"{what}: rank {r} rows [{rb},{re}) of layer {l}"
            assert out[:rb].isnan().all() and out[re:].isnan().all(), f"{what}: rank {r} wrote outside its rows (layer {l})"
            gathered[rb:re] = out[rb:re]
            if last:
                assert torch.equal(sc[rb:re], ref_score[rb:re]), f"{what}: rank {r} scores"
                assert sc[:rb].isnan().all() and sc[re:].isnan().all(), f"{what}: rank {r} wrote scores outside its rows"
                score[rb:re] = sc[rb:re]
        h = gathered
        hs.append(h)
    assert torch.equal(h, ref_h[-1]) and torch.equal(score, ref_score), what
    return hs, score


@pytest.mark.parametrize("F", [32, 64, 128])
@pytest.mark.parametrize("algo", ["umma", "umma2", "ffma"])
@pytest.mark.parametrize("family", ["hub_src", "hub_dst", "trace", "trace_aligned"])
def test_sharded_forward_matches_single_gpu(family, algo, F):
    """Every (world, cut, rowptr type, edge-block placement) of one graph family and kernel path."""
    name, align = family_graph(family)
    rp, col, ew, x_np = graph(name, F)
    models = make_models(F, algo, 9)
    x = torch.from_numpy(x_np).cuda()
    misaligned_base = False
    for rp64 in (False, True):
        rph = rp.astype(np.int64) if rp64 else rp
        ref = single_gpu(models[-1], x, *(torch.from_numpy(a).cuda() for a in (rph, col, ew)))
        for world in (2, 3, 8):
            for cut in ("edges", "rows"):
                for source in ("host", "device", "offset"):
                    what = f"{family} {algo} F={F} rowptr{64 if rp64 else 32} world={world} cut={cut} {source}"
                    shards = make_shards(rph, col, ew, world, source, cut=cut, align=align)
                    assert shards[0].cuts[0] == 0 and shards[0].cuts[-1] == x.shape[0]
                    if source == "host":
                        misaligned_base |= any(sh.edge_base % 4 for sh in shards)
                    hs, score = emulate_allgather(models[:world], shards, x, ref, what)
    if wants_oracle(name, algo, F):
        check_oracle(name, F, algo, hs, score, what)
    assert misaligned_base, "no shard had an edge block starting off a 16-byte boundary"


def row_split_edge_cuts(rowptr):
    """Cuts with an empty rank at the start and one in the middle, ranks of 7 and 13 rows, row_begin off the 32-row
    tile grid, and cuts directly before and directly after one hub row (a rank holding only that row)."""
    hubs = np.flatnonzero(np.diff(rowptr) > LONG_T)
    h = int(hubs[hubs.size // 2])
    assert h > 21 and np.diff(rowptr)[h] > LONG_T
    return [0, 0, 7, 20, 20, h, h + 1, rowptr.size - 1]


@pytest.mark.parametrize("algo", ["umma", "umma2", "ffma"])
@pytest.mark.parametrize("family", ["hub_dst", "trace"])
def test_sharded_forward_row_split_edges(family, algo, monkeypatch):
    for F in (32, 128):
        rp, col, ew, x_np = graph(family, F)
        cuts = row_split_edge_cuts(rp)
        world = len(cuts) - 1
        models = make_models(F, algo, world + 1)
        x = torch.from_numpy(x_np).cuda()
        for rp64 in (False, True):
            rph = rp.astype(np.int64) if rp64 else rp
            ref = single_gpu(models[-1], x, *(torch.from_numpy(a).cuda() for a in (rph, col, ew)))
            for source in ("host", "offset"):
                what = f"{family} {algo} F={F} rowptr{64 if rp64 else 32} cuts={cuts} {source}"
                shards = make_shards(rph, col, ew, world, source, cuts=cuts, monkeypatch=monkeypatch)
                hs, score = emulate_allgather(models[:world], shards, x, ref, what)
        if wants_oracle(family, algo, F):
            check_oracle(family, F, algo, hs, score, what)


# ----------------------------------------------------------------------------------------------- 2. fused peer stores
def emulate_peer_stores(models, shards, x, ref, masks, what):
    """Sharded forward with the exchange fused into the epilogue: every rank has two NaN-filled [N, H] buffers; a layer
    other than the last stores each produced row into the rank's own buffer and into the other ranks' buffers of the
    same parity (slot order), only where the need bit is set when masks are given.  After each such layer, every
    buffer must hold exactly the rows it was sent."""
    ref_h, ref_score = ref
    N, world = x.shape[0], len(shards)
    layer = [D.cuda_layer_fn(m) for m in models]
    bufs = [[torch.full((N, H), NAN, device="cuda") for _ in range(2)] for _ in range(world)]
    scores = [torch.full((N,), NAN, device="cuda") for _ in range(world)]
    need = [torch.from_numpy(m).cuda() for m in masks] if masks is not None else None
    h_in = [x] * world
    for l in range(LAYERS):
        last = l == LAYERS - 1
        for r in range(world):
            bufs[r][l & 1].fill_(NAN)
        for r, sh in enumerate(shards):
            peers = None if last else [bufs[p][l & 1] for p in range(world) if p != r]
            layer[r](l, h_in[r], bufs[r][l & 1], sh, score_out=scores[r] if last else None, peer_outs=peers,
                     peer_need=need[r] if need is not None and not last else None)
        for r, sh in enumerate(shards):
            own = slice(sh.row_begin, sh.row_end)
            assert torch.equal(bufs[r][l & 1][own], ref_h[l][own]), f"{what}: rank {r} own rows of layer {l}"
        if not last:
            for p in range(world):
                want = torch.full((N, H), NAN, device="cuda")
                for r, sh in enumerate(shards):
                    rows = torch.arange(sh.row_begin, sh.row_end, device="cuda")
                    if r != p and need is not None:
                        slot = p - (p > r)
                        rows = rows[((need[r][rows] >> slot) & 1).bool()]
                    want[rows] = bufs[r][l & 1][rows]
                got = bufs[p][l & 1]
                bad = (bits(got) != bits(want)).any(1)
                assert not bad.any(), (f"{what}: layer {l}, rank {p}'s buffer: {int(bad.sum())} rows differ from the rows "
                                       f"it was sent, first {bad.nonzero()[:8, 0].tolist()}")
        h_in = [bufs[r][l & 1] for r in range(world)]
    for r, sh in enumerate(shards):
        own = slice(sh.row_begin, sh.row_end)
        assert torch.equal(scores[r][own], ref_score[own]), f"{what}: rank {r} scores"


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("algo", ["umma", "umma2"])
@pytest.mark.parametrize("family,F", [("hub_src", 32), ("hub_dst", 128), ("trace", 64)])
def test_fused_peer_stores(family, F, algo, world):
    rp, col, ew, x_np = graph(family, F)
    models = make_models(F, algo, world + 1)
    x = torch.from_numpy(x_np).cuda()
    ref = single_gpu(models[-1], x, *(torch.from_numpy(a).cuda() for a in (rp, col, ew)))
    shards = make_shards(rp, col, ew, world, "host")
    masks = need_masks(rp, col, shards[0].cuts)
    assert any((m != 0).any() for m in masks) and any((m != (1 << (world - 1)) - 1).any() for m in masks)
    for use_mask in (True, False):
        emulate_peer_stores(models[:world], shards, x, ref, masks if use_mask else None,
                            f"{family} {algo} F={F} world={world} {'need mask' if use_mask else 'every row'}")


def test_peer_arguments_are_checked():
    """n_peers above the 7 the epilogue holds, peers with the fp32 layer and a NULL peer_out are refused before any
    launch; 7 peers run and every peer buffer receives every row."""
    N = 700
    g = G.synthetic_graph(N=N, E=9000, seed=8)
    model = GraphSAGE_T(32, H, 1).cuda()
    x, rp, col, ew = (torch.from_numpy(a).cuda() for a in (g.x, g.rowptr, g.col, g.ew))
    out = torch.full((N, H), NAN, device="cuda")
    peers = [torch.full((N, H), NAN, device="cuda") for _ in range(8)]

    def call(algo, peer_out, n_peers):
        L.check(L.lib().nerrf_sage_layer_fwd_ex(
            L.ptr(x), L.ptr(rp), 0, L.ptr(col), L.ptr(ew), L.ptr(model.weights[0]), L.ptr(model.biases[0]), L.ptr(out), N,
            0, N, 32, H, 1, ALGO_CODE[algo], None, 0.0, None, None, 0, peer_out, n_peers, None, L.current_stream_ptr()),
            "nerrf_sage_layer_fwd_ex")

    with pytest.raises(L.NerrfError):
        call("umma", L.ptr_array(peers), 8)
    with pytest.raises(L.NerrfError):
        call("ffma", L.ptr_array(peers[:1]), 1)
    with pytest.raises(L.NerrfError):
        call("umma", None, 1)
    assert out.isnan().all() and all(p.isnan().all() for p in peers)
    call("umma", L.ptr_array(peers[:7]), 7)
    assert torch.equal(out, model.layer_forward(0, x, rp, col, ew))
    assert all(torch.equal(p, out) for p in peers[:7]) and peers[7].isnan().all()


# ----------------------------------------------------------------------------------------------- 3. hub rows
@pytest.mark.parametrize("F", [32, 64, 128])
@pytest.mark.parametrize("algo", ["umma", "umma2", "ffma"])
def test_row_ranges_through_hub_rows(algo, F):
    """Ranges that start and end inside the run of hub rows of a hub_dst graph, under ONE model: bit-equal to the
    full-range layer, nothing written outside; the second layer with the hub-row scan reused equals a fresh scan."""
    rp_np, col_np, ew_np, x_np = graph("hub_dst", F)
    deg = np.diff(rp_np)
    hub_end = int(np.argmax(deg <= LONG_T))
    assert hub_end > 150 and (deg[:hub_end] > LONG_T).all()
    x, rp, col, ew = (torch.from_numpy(a).cuda() for a in (x_np, rp_np, col_np, ew_np))
    ref_model, model = make_models(F, algo, 2)
    h0 = ref_model.layer_forward(0, x, rp, col, ew)
    h1 = ref_model.layer_forward(1, h0, rp, col, ew)
    lin = ref_model.layer_forward(0, x, rp, col, ew, relu=False)          # the epilogue's no-ReLU branch
    W, b = ref_model.oracle_params()["layers"][0]
    t = torch.from_numpy
    assert (lin < 0).any()
    assert_close_fp32(lin, S.layer(t(x_np), t(rp_np), t(col_np), t(ew_np), W, b, relu=False, dtype=torch.float64),
                      atol_rms=ATOL_RMS[algo], what=f"{algo} F={F} relu=False vs fp64 oracle")
    N = x.shape[0]
    for rb, re in [(3, 45), (40, 41), (17, hub_end - 1), (1, 2), (hub_end - 40, hub_end - 3)]:
        assert deg[rb - 1] > LONG_T and deg[rb] > LONG_T and deg[re - 1] > LONG_T
        outs = []
        for l, h, reuse, relu in [(0, x, False, True), (1, h0, True, True), (1, h0, False, True), (0, x, False, False)]:
            out = torch.full((N, H), -7.0, device="cuda")
            model.layer_forward(l, h, rp, col, ew, out=out, row_begin=rb, row_end=re, relu=relu, reuse_long_scan=reuse)
            assert (out[:rb] == -7).all() and (out[re:] == -7).all(), f"rows outside [{rb},{re}) written"
            outs.append(out[rb:re])
        assert torch.equal(outs[0], h0[rb:re]), f"{algo} F={F} layer 1 rows [{rb},{re})"
        assert torch.equal(outs[1], h1[rb:re]), f"{algo} F={F} layer 2 rows [{rb},{re}), hub-row scan reused"
        assert torch.equal(outs[2], h1[rb:re]), f"{algo} F={F} layer 2 rows [{rb},{re}), fresh hub-row scan"
        assert torch.equal(outs[3], lin[rb:re]), f"{algo} F={F} layer 1 rows [{rb},{re}) without ReLU"


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


@pytest.mark.parametrize("F", [32, 128])
@pytest.mark.parametrize("algo", ["umma", "umma2"])
def test_hub_row_scratch_smaller_than_the_graph_needs(algo, F):
    """A scratch with room for a few chunk items: the hub rows that fit are pre-aggregated, the others stay inline.
    The result is within the oracle bound and close to the inline-only call; a scratch below the 8 KB minimum is not
    used at all (bit-equal to the call without one)."""
    rp_np, col_np, ew_np, x_np = graph("hub_dst", F)
    deg = np.diff(rp_np).astype(np.int64)
    nbytes = 8192 + 64
    cap = long_ws_capacity(nbytes)
    assert 4 <= cap <= 16
    rb = int(np.flatnonzero(-(-deg // LONG_CH) > cap).max()) + 1        # every hub row from rb on fits on its own
    N = x_np.shape[0]
    hub = deg[rb:] > LONG_T
    items = int((-(-deg[rb:][hub] // LONG_CH)).sum())
    assert items > 4 * cap, f"the rows need {items} chunk items, the scratch holds {cap}"
    x, rp, col, ew = (torch.from_numpy(a).cuda() for a in (x_np, rp_np, col_np, ew_np))
    model = make_models(F, algo, 1)[0]

    def layer(ws, nb):
        out = torch.full((N, H), -7.0, device="cuda")
        L.check(L.lib().nerrf_sage_layer_fwd_ex(
            L.ptr(x), L.ptr(rp), 0, L.ptr(col), L.ptr(ew), L.ptr(model.weights[0]), L.ptr(model.biases[0]), L.ptr(out), N,
            rb, N, F, H, 1, ALGO_CODE[algo], None, 0.0, None, L.ptr(ws), nb, None, 0, None, L.current_stream_ptr()),
            "nerrf_sage_layer_fwd_ex")
        assert (out[:rb] == -7).all()
        return out[rb:]

    inline = layer(None, 0)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    some = layer(ws, nbytes)
    assert int(ws[:4].view(torch.int32)) == items, "the scan did not claim one item per chunk of every hub row"
    W, b = model.oracle_params()["layers"][0]
    t = torch.from_numpy
    want = S.layer(t(x_np), t(rp_np), t(col_np), t(ew_np), W, b, row_begin=rb, dtype=torch.float64)
    assert_close_fp32(some, want, atol_rms=ATOL_RMS[algo], what=f"{algo} F={F} partial scratch vs fp64 oracle")
    assert_close_fp32(some, inline, atol_rms=ATOL_RMS[algo], what=f"{algo} F={F} partial scratch vs inline")
    assert torch.equal(layer(torch.zeros(8191, dtype=torch.uint8, device="cuda"), 8191), inline)
