"""Tensor-core GraphSAGE-T layer at F = 64 / 128, where a prep kernel computes the self half x_v . W[0:F] into the
output rows and the layer kernel finishes the mean half from there (needs an H100): stale output contents, isolated rows
and tiles, row ranges off the tile grid, hub rows, and parity with the oracle."""
import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G
from nerrf_b200.ai.models import GraphSAGE_T
from oracle import sage_ref as S
from gpu_util import ATOL_RMS, dev_graph, cpu_graph, assert_close_fp32

pytestmark = pytest.mark.gpu

N = 1000
ISOLATED = range(101, 197)          # contains a whole 32-row tile for row_begin 0 and for row_begin 37
LONE = (range(300, 400), 350)       # rows without in-edges except one, in a tile of their own for both row_begins


def _graph(F, hub, seed):
    """Random rows, scattered and tiled isolated rows, and one row of 600 (hub) or 60 in-edges among isolated ones."""
    rng = np.random.default_rng(seed)
    E = 12000
    dst = rng.integers(0, N, E)
    scattered = rng.choice(N, N // 10, replace=False)                             # 10 % of the rows stay isolated
    dst = dst[~np.isin(dst, np.r_[ISOLATED, LONE[0], scattered])]
    deg = 600 if hub else 60
    dst = np.concatenate([dst, np.full(deg, LONE[1]), np.full(deg, 7)])         # row 7: a second long row
    src = rng.integers(0, N, dst.size)
    t = (rng.random(dst.size) * 60).astype(np.float32); conf = (0.5 + 0.5 * rng.random(dst.size)).astype(np.float32)
    rowptr, col, ew = G.csr_from_edges(src, dst, t, conf, N)
    d = np.diff(rowptr)
    assert (d[list(ISOLATED)] == 0).all() and d[LONE[1]] == deg and (d == 0).sum() > len(ISOLATED) + 99
    return G.TemporalGraph(rowptr, col, ew, rng.standard_normal((N, F)).astype(np.float32), {})


@pytest.mark.parametrize("algo", ["umma", "umma2"])
@pytest.mark.parametrize("F", [64, 128])
@pytest.mark.parametrize("rowptr64", [False, True])
@pytest.mark.parametrize("hub", [False, True])
def test_self_split_layer(algo, F, rowptr64, hub):
    g = _graph(F, hub, seed=F + hub)
    model = GraphSAGE_T(F, 128, 1, algo=algo).cuda()
    W, b = model.oracle_params()["layers"][0]
    x, rp, col, ew = dev_graph(g, rowptr64=rowptr64)
    node_w = model.node_w.detach().double().cpu()
    node_b = float(model.node_b.detach())
    for relu in (True, False):
        for head in (False, True):
            full = torch.zeros(N, 128, device="cuda")
            sc_full = torch.zeros(N, device="cuda")
            model.layer_forward(0, x, rp, col, ew, out=full, relu=relu, score_out=sc_full if head else None)
            want = S.layer(*cpu_graph(g), W, b, relu=relu)
            what = f"{algo} F={F} rowptr64={rowptr64} hub={hub} relu={relu} head={head}"
            assert_close_fp32(full, want, atol_rms=ATOL_RMS[algo], what=what)
            if head:
                want_sc = torch.sigmoid(want.double() @ node_w + node_b)
                assert float((sc_full.cpu().double() - want_sc).abs().max()) < 1e-5, what
            # the result does not depend on what out held, and only [row_begin, row_end) is written
            for rb, re in ((0, N), (37, N - 45), (5, 20), (350, 351)):
                for fill in (float("nan"), 0.0, -7.0):
                    out = torch.full((N, 128), fill, device="cuda")
                    sc = torch.full((N,), fill, device="cuda")
                    model.layer_forward(0, x, rp, col, ew, out=out, row_begin=rb, row_end=re, relu=relu,
                                        score_out=sc if head else None)
                    assert torch.equal(out[rb:re], full[rb:re]), f"{what} rows [{rb},{re}) fill {fill}"
                    outside = torch.cat([out[:rb], out[re:]])
                    assert (outside.isnan().all() if fill != fill else (outside == fill).all()), f"{what} [{rb},{re}) fill {fill}"
                    if head:
                        assert torch.equal(sc[rb:re], sc_full[rb:re]), what
                        sc_out = torch.cat([sc[:rb], sc[re:]])
                        assert (sc_out.isnan().all() if fill != fill else (sc_out == fill).all()), what
            # isolated rows: bias only (then ReLU), exactly as the oracle's zero mean gives
            iso = torch.from_numpy(np.diff(g.rowptr) == 0)
            assert iso[list(ISOLATED)].all()
            assert_close_fp32(full.cpu()[iso], want[iso], atol_rms=ATOL_RMS[algo], what=what + " isolated rows")
