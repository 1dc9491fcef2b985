"""The F = 64 / 128 tensor-core GraphSAGE-T layer (needs an H100) in both its shapes: at F = 128 without hub rows the split
mean-half weights resident in the consumer registers and each tile pair's MMAs in one wgmma commit group; at F = 64 and
with hub rows the fragments read from L2 one K step ahead.  Fewer tiles than SMs, a single partial tile, rows without
in-edges, odd tile counts (a pass that ends on the closing entry), row ranges off the 32-row grid, hub destinations (the
hub-row partial items) and int64 row pointers, at NS = 3 ("umma") and NS = 2 ("umma2"), with and without the fused node
head.  Each result is checked against the fp32 CUDA-core layer ("ffma") and the oracle, and must be bit-equal across
launches; a 1-layer model, whose only layer carries the fused head, is checked end to end."""
import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G
from nerrf_b200.ai.models import GraphSAGE_T
from oracle import sage_ref as S
from gpu_util import ATOL_RMS, dev_graph, cpu_graph, assert_close_fp32

pytestmark = pytest.mark.gpu


def _graph(n, F, seed, isolated=0.0, hub=False):
    rng = np.random.default_rng(seed)
    dst = rng.integers(0, n, 8 * n)
    if isolated:                                              # rows with no in-edges at all
        dst = dst[~np.isin(dst, rng.choice(n, max(1, int(n * isolated)), replace=False))]
    if hub:                                                   # hub destinations: rows far above the 128-edge threshold
        hubs = rng.choice(n, max(1, n // 64), replace=False)
        dst = np.concatenate([dst, np.repeat(hubs, 300)])
    src = rng.integers(0, n, dst.size)
    t = (rng.random(dst.size) * 60).astype(np.float32)
    conf = (0.5 + 0.5 * rng.random(dst.size)).astype(np.float32)
    rowptr, col, ew = G.csr_from_edges(src, dst, t, conf, n)
    return G.TemporalGraph(rowptr, col, ew, rng.standard_normal((n, F)).astype(np.float32), {})


def _layer(model, dg, n, rb, re, relu, head):
    x, rp, col, ew = dg
    out = torch.full((n, 128), float("nan"), device="cuda")
    sc = torch.full((n,), float("nan"), device="cuda")
    model.layer_forward(0, x, rp, col, ew, out=out, row_begin=rb, row_end=re, relu=relu, score_out=sc if head else None)
    torch.cuda.synchronize()
    return out, sc


def _check(g, F, algo, rb, re, what, rowptr64=False):
    model = GraphSAGE_T(F, 128, 1, algo=algo).cuda()
    ffma = GraphSAGE_T(F, 128, 1, algo="ffma").cuda()
    W, b = model.oracle_params()["layers"][0]
    dg = dev_graph(g, rowptr64=rowptr64)
    n = g.x.shape[0]
    for relu in (True, False):
        want = S.layer(*cpu_graph(g), W, b, relu=relu)[rb:re]
        for head in (False, True):
            tag = f"{what} relu={relu} head={head} rows [{rb},{re})"
            out, sc = _layer(model, dg, n, rb, re, relu, head)
            assert_close_fp32(out[rb:re], want, atol_rms=ATOL_RMS[algo], what=tag + " vs oracle")
            assert torch.cat([out[:rb], out[re:]]).isnan().all(), tag
            ref, ref_sc = _layer(ffma, dg, n, rb, re, relu, head)
            assert_close_fp32(out[rb:re], ref[rb:re], atol_rms=ATOL_RMS[algo], what=tag + " vs ffma")
            again, again_sc = _layer(model, dg, n, rb, re, relu, head)
            assert torch.equal(out[rb:re], again[rb:re]), tag + ": not bit-equal across launches"
            if head:
                assert float((sc[rb:re] - ref_sc[rb:re]).abs().max()) < 1e-5, tag
                assert torch.equal(sc[rb:re], again_sc[rb:re]), tag + ": scores not bit-equal across launches"


@pytest.mark.parametrize("algo", ["umma", "umma2"])
@pytest.mark.parametrize("F", [64, 128])
@pytest.mark.parametrize("tiles", [1, 5, 133, 266])
def test_f128_resident(F, algo, tiles):
    n = 32 * tiles - 7                                        # the last tile is partial (tiles = 1: the only tile)
    g = _graph(n, F, seed=tiles, isolated=0.1)
    assert (np.diff(g.rowptr) == 0).any()
    _check(g, F, algo, 0, n, f"F={F} {algo} tiles={tiles}")
    if tiles >= 5:                                            # a row range that starts and ends off the 32-row grid
        _check(g, F, algo, 13, n - 21, f"F={F} {algo} tiles={tiles}")


@pytest.mark.parametrize("rowptr64", [False, True])
@pytest.mark.parametrize("algo", ["umma", "umma2"])
@pytest.mark.parametrize("F", [64, 128])
def test_f128_resident_hub_destinations(F, algo, rowptr64):
    n = 32 * 265 - 7
    g = _graph(n, F, seed=3, hub=True)
    assert np.diff(g.rowptr).max() > 256
    _check(g, F, algo, 0, n, f"F={F} {algo} hub destinations rowptr64={rowptr64}", rowptr64=rowptr64)
    _check(g, F, algo, 45, n - 3, f"F={F} {algo} hub destinations rowptr64={rowptr64}", rowptr64=rowptr64)


@pytest.mark.parametrize("algo", ["umma", "umma2"])
@pytest.mark.parametrize("F", [64, 128])
def test_f128_resident_one_layer_model(F, algo):
    """A 1-layer model: its only layer is the F = 64 / 128 one, with the fused node head."""
    g = _graph(32 * 140 + 5, F, seed=11, isolated=0.05)
    model = GraphSAGE_T(F, 128, 1, algo=algo).cuda()
    ffma = GraphSAGE_T(F, 128, 1, algo="ffma").cuda()
    h, sc = model(*dev_graph(g))
    h2, sc2 = model(*dev_graph(g))
    hf, scf = ffma(*dev_graph(g))
    hw, scw = S.forward(model.oracle_params(), *cpu_graph(g))
    assert_close_fp32(h, hw, atol_rms=ATOL_RMS[algo], what=f"F={F} {algo} 1-layer model vs oracle")
    assert_close_fp32(h, hf, atol_rms=ATOL_RMS[algo], what=f"F={F} {algo} 1-layer model vs ffma")
    assert float((sc.cpu() - scw).abs().max()) < 1e-5
    assert float((sc - scf).abs().max()) < 1e-5
    assert torch.equal(h, h2) and torch.equal(sc, sc2)
