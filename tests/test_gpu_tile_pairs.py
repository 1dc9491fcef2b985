"""Tile pairs in the F = 64 / 128 tensor-core GraphSAGE-T layer (needs an H100): each consumer warpgroup runs the CTA's
tiles two at a time from one weight-fragment load.  Tile counts that end a CTA's stream on either slot of a pair, row
ranges off the 32-row grid, the fused head, relu off and hub-destination rows; every result is bit-equal across repeated
launches (the dynamic schedule pairs different tiles each time) and within tolerance of the oracle."""
import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G
from nerrf_b200.ai.models import GraphSAGE_T
from oracle import sage_ref as S
from gpu_util import ATOL_RMS, dev_graph, cpu_graph, assert_close_fp32

pytestmark = pytest.mark.gpu

REPEATS = 5


def _graph(n, F, seed, hub=False):
    rng = np.random.default_rng(seed)
    dst = rng.integers(0, n, 8 * n)
    if hub:                                                   # hub destinations: rows far above the 128-edge threshold
        hubs = rng.choice(n, max(1, n // 64), replace=False)
        dst = np.concatenate([dst, np.repeat(hubs, 300)])
    src = rng.integers(0, n, dst.size)
    t = (rng.random(dst.size) * 60).astype(np.float32)
    conf = (0.5 + 0.5 * rng.random(dst.size)).astype(np.float32)
    rowptr, col, ew = G.csr_from_edges(src, dst, t, conf, n)
    return G.TemporalGraph(rowptr, col, ew, rng.standard_normal((n, F)).astype(np.float32), {})


def _check(g, F, algo, rb, re, what):
    model = GraphSAGE_T(F, 128, 1, algo=algo).cuda()
    W, b = model.oracle_params()["layers"][0]
    node_w = model.node_w.detach().double().cpu()
    node_b = float(model.node_b.detach())
    x, rp, col, ew = dev_graph(g)
    n = g.x.shape[0]
    for relu in (True, False):
        want = S.layer(*cpu_graph(g), W, b, relu=relu)[rb:re]
        for head in (False, True):
            tag = f"{what} relu={relu} head={head} rows [{rb},{re})"
            first = first_sc = None
            for _ in range(REPEATS):
                out = torch.full((n, 128), float("nan"), device="cuda")
                sc = torch.full((n,), float("nan"), device="cuda")
                model.layer_forward(0, x, rp, col, ew, out=out, row_begin=rb, row_end=re, relu=relu,
                                    score_out=sc if head else None)
                if first is None:
                    first, first_sc = out.clone(), sc.clone()
                    assert_close_fp32(out[rb:re], want, atol_rms=ATOL_RMS[algo], what=tag)
                    assert torch.cat([out[:rb], out[re:]]).isnan().all(), tag
                    if head:
                        want_sc = torch.sigmoid(want.double() @ node_w + node_b)
                        assert float((sc[rb:re].cpu().double() - want_sc).abs().max()) < 1e-5, tag
                else:
                    assert torch.equal(out[rb:re], first[rb:re]), tag + ": not bit-equal across launches"
                    if head:
                        assert torch.equal(sc[rb:re], first_sc[rb:re]), tag + ": scores not bit-equal across launches"


@pytest.mark.parametrize("algo", ["umma", "umma2"])
@pytest.mark.parametrize("F", [64, 128])
@pytest.mark.parametrize("tiles", [1, 2, 3, 133, 265])
def test_tile_pairs(algo, F, tiles):
    n = 32 * tiles - 7                                        # the last tile is partial
    g = _graph(n, F, seed=tiles + F)
    _check(g, F, algo, 0, n, f"{algo} F={F} tiles={tiles}")
    if tiles >= 3:                                            # a row range that starts and ends off the 32-row grid
        _check(g, F, algo, 13, n - 21, f"{algo} F={F} tiles={tiles}")


@pytest.mark.parametrize("algo", ["umma", "umma2"])
@pytest.mark.parametrize("F", [64, 128])
def test_tile_pairs_hub_destinations(algo, F):
    n = 32 * 265 - 7
    g = _graph(n, F, seed=F + 1, hub=True)
    assert np.diff(g.rowptr).max() > 256
    _check(g, F, algo, 0, n, f"{algo} F={F} hub destinations")
    _check(g, F, algo, 45, n - 3, f"{algo} F={F} hub destinations")
