"""L2 eviction-priority hints of the tensor-core GraphSAGE-T layer (NERRF_SAGE_FLAG_NO_L2_POLICY to turn them off).

Hints only change which lines L2 evicts first, so every output must be the same bits with the policy on and off: layer
by layer (int32 and int64 rowptr, row ranges off the tile grid, edge blocks passed alone), the whole forward and the
host session, on hub-source, hub-destination (long-row path), uniform and trace-structured graphs."""
import functools

import numpy as np
import pytest
import torch

from nerrf_b200 import dist as D, graph as G
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.ai.models.graphsage_t import HostSession

pytestmark = pytest.mark.gpu

H, LAYERS = 128, 3
N_SYN, E_SYN = 24_000, 360_000


@functools.lru_cache(maxsize=None)
def graph(family, F):
    """(rowptr int32, col, ew, x [N, F]) as host arrays."""
    if family == "trace":
        rp, col, ew, _, _ = D.gpu_trace_graph(500, "cuda")
    elif family == "uniform":
        rp, col, ew, _ = D.gpu_synthetic_graph(N_SYN, E_SYN, 5, "cuda", family="uniform")
    else:
        g = G.synthetic_graph(N=N_SYN, E=E_SYN, seed=3, hub=family[4:], f_in=F)
        return g.rowptr, g.col, g.ew, g.x
    rp, col, ew = (t.cpu().numpy() for t in (rp, col, ew))
    return rp.astype(np.int32), col, ew, np.random.default_rng(F).standard_normal((rp.size - 1, F), dtype=np.float32)


def dev(rp, col, ew, x, rowptr64=False):
    return (torch.from_numpy(rp.astype(np.int64 if rowptr64 else np.int32)).cuda(), torch.from_numpy(col).cuda(),
            torch.from_numpy(ew).cuda(), torch.from_numpy(x).cuda())


def model_pair(F):
    on = GraphSAGE_T(F, H, LAYERS).cuda()
    off = GraphSAGE_T(F, H, LAYERS).cuda().load_oracle_params(on.oracle_params())
    off.l2_policy = False
    return on, off


def layers(model, x, rp, col, ew, **kw):
    """The forward layer by layer (layers 2.. reuse the graph scan) -> ([h_1 .. h_L], score)."""
    N = x.shape[0]
    outs, h = [], x
    score = torch.full((N,), float("nan"), device="cuda")
    for l in range(LAYERS):
        out = torch.full((N, H), float("nan"), device="cuda")
        h = model.layer_forward(l, h, rp, col, ew, out=out, score_out=score if l == LAYERS - 1 else None,
                                reuse_long_scan=l > 0, **kw)
        outs.append(h)
    return outs, score


def assert_same_bits(a, b, what):
    a, b = a.cpu(), b.cpu()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"{what}: policy on and off differ"


# ----------------------------------------------------------------------------------------------- bit equality
@pytest.mark.parametrize("F", [32, 64, 128])
@pytest.mark.parametrize("family", ["hub_src", "hub_dst", "uniform", "trace"])
def test_layers_same_bits_on_and_off(F, family):
    rp, col, ew, x = dev(*graph(family, F))
    on, off = model_pair(F)
    (h_on, s_on), (h_off, s_off) = layers(on, x, rp, col, ew), layers(off, x, rp, col, ew)
    for l in range(LAYERS):
        assert_same_bits(h_on[l], h_off[l], f"{family} F={F} layer {l + 1}")
    assert_same_bits(s_on, s_off, f"{family} F={F} fused head")


@pytest.mark.parametrize("rowptr64", [False, True])
@pytest.mark.parametrize("F", [32, 128])
def test_row_range_and_edge_block(F, rowptr64):
    """A row range off the tile grid whose edge block is passed alone (edge_base), as a shard of a sharded forward."""
    rph, colh, ewh, xh = graph("hub_src", F)
    rb, re = 1_005, N_SYN - 3_007
    e0, e1 = int(rph[rb]), int(rph[re])
    rp, _, _, x = dev(rph, colh, ewh, xh, rowptr64)
    col, ew = torch.from_numpy(colh[e0:e1].copy()).cuda(), torch.from_numpy(ewh[e0:e1].copy()).cuda()
    on, off = model_pair(F)
    kw = dict(row_begin=rb, row_end=re, edge_base=e0)
    (h_on, s_on), (h_off, s_off) = layers(on, x, rp, col, ew, **kw), layers(off, x, rp, col, ew, **kw)
    for l in range(LAYERS):
        assert_same_bits(h_on[l], h_off[l], f"shard F={F} layer {l + 1}")
    assert_same_bits(s_on, s_off, f"shard F={F} head")


@pytest.mark.parametrize("family", ["hub_src", "hub_dst"])
def test_forward_same_bits(family):
    rp, col, ew, x = dev(*graph(family, 32))
    on, off = model_pair(32)
    h_on, s_on = on(x, rp, col, ew)
    h_off, s_off = off(x, rp, col, ew)
    assert_same_bits(h_on, h_off, f"{family} forward")
    assert_same_bits(s_on, s_off, f"{family} forward scores")


def test_host_session_same_bits():
    """Large enough for the session's chunked layer 1 (four row ranges, each with its own edge block)."""
    g = G.synthetic_graph(N=100_000, E=1_200_000, seed=4)
    on, off = model_pair(32)
    res = []
    for m in (on, off):
        s = HostSession(m, g.num_nodes, g.num_edges)
        score = torch.empty(g.num_nodes)
        h = torch.empty(g.num_nodes, H)
        s.forward(*(torch.from_numpy(a) for a in (g.x, g.rowptr, g.col, g.ew)), score, h)
        res.append((h, score))
        s.close()
    assert_same_bits(res[0][0], res[1][0], "session h")
    assert_same_bits(res[0][1], res[1][1], "session scores")
