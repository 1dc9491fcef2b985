"""BASELINE config 5 in miniature (needs an H100): a fleet trace streamed tick by tick through the sliding window, the
GPU graph constructor, GraphSAGE_T, the LSTM on the top-A candidates and the MCTS planner with process-kill candidates
(planner spec v1) -- the running undo plan must end up reverting the encrypted files and killing their writers."""
import numpy as np
import pytest
import torch

from nerrf_b200 import stream
from nerrf_b200.ai import train as T
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.ai.models.lstm import LSTMScorer

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def models():
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3)
    return model.cuda(), scorer.cuda()


@pytest.mark.parametrize("kills", [False, True])
def test_streamed_fleet_trace_plans_the_reversions(models, kills):
    model, scorer = models
    cols, enc, bad = stream.fleet_columns(120, 5, seed=9, return_pids=True)
    sp = stream.StreamingPlanner(model, scorer, top_a=1024, n_rollouts=512, depth=24, iterations=8, commit_per_search=32,
                                 kill_candidates=kills)
    ticks = sp.run(cols)
    assert len(ticks) >= 3 and ticks[0].planned == []            # nothing is encrypted in the first 30 s
    planned = set(sp.reverted)
    tp = len(planned & enc)
    assert tp / len(enc) >= 0.95, (tp, len(enc))                  # recall: (nearly) every encrypted file is renamed back
    assert tp / max(len(planned), 1) >= 0.90                      # precision: the ransom note is the usual extra
    assert all(t.timings_ms["graphsage_t"] > 0 and "sequences" in t.timings_ms for t in ticks if t.planned)
    if kills:
        assert sp.killed and sp.killed <= bad                     # only ransomware processes are killed ...
        assert len(sp.killed) >= len(bad) - 1                     # ... and (nearly) all of them
    else:
        assert not sp.killed


def test_device_stream_window_equals_the_columnar_constructor():
    """stream.DeviceStream.window_graph (columns resident in HBM, interning + features + edges + CSR on the GPU) builds
    the same graph as ingest.graph_from_columns over stream.window(...): node numbering, CSR, labels, names, name hashes;
    sequences of a node subset equal ingest.sequences_from_columns."""
    from nerrf_b200 import ingest
    cols, enc = stream.fleet_columns(60, 4, seed=3)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    for (lo, hi) in [(t0 - 1, t0 + 30), (t0 + 10, t0 + 70), (t0 + 40, t1), (t1 + 5, t1 + 9)]:
        g = ds.window_graph(lo, hi, 60.0)
        w = stream.window(cols, lo, hi)
        if w.n == 0:
            assert g is None
            continue
        want = ingest.graph_from_columns(w, device="cuda", observable=True, window=60.0)
        assert g.num_nodes == want.num_nodes and torch.equal(g.rowptr, want.rowptr) and torch.equal(g.col, want.col)
        assert torch.allclose(g.ew, want.ew, rtol=1e-6, atol=0) and torch.allclose(g.x, want.x, rtol=1e-6, atol=1e-7)
        assert np.array_equal(g.meta["label"], want.meta["label"]) and np.array_equal(g.meta["node_kind"], want.meta["node_kind"])
        assert np.allclose(g.meta["size_mb"], want.meta["size_mb"])
        names = g.meta["names"]
        pick = np.random.default_rng(0).integers(0, g.num_nodes, 200)
        assert [names[int(v)] for v in pick] == [want.meta["names"][int(v)] for v in pick]
        nh = g.meta["name_hash"].cpu().numpy()
        assert all(int(nh[int(v)]) == stream.name_hash(names[int(v)]) for v in pick[:50])
        files = np.nonzero(g.meta["node_kind"] == 0)[0][::7]
        sq, ln, have = ds.sequences(g, files)
        sq2, ln2, have2 = ingest.sequences_from_columns(w, observable=True, only_nodes=files)
        assert np.array_equal(have, have2) and np.array_equal(ln, ln2) and np.array_equal(sq, sq2)
        # the same sequences built on the device from the resident columns (any candidate order, duplicates allowed)
        pick_f = np.random.default_rng(1).permutation(have)[:200]
        sq_d, ln_d = ds.sequences_device(g, pick_f)
        pos = np.searchsorted(have, pick_f)
        assert np.array_equal(ln_d.cpu().numpy(), ln[pos])
        assert np.allclose(sq_d.cpu().numpy(), sq[pos], rtol=1e-6, atol=1e-7)
        assert np.array_equal(sq_d.cpu().numpy()[:, :, :8], sq[pos][:, :, :8])           # one-hot slots exactly


def test_empty_stream_is_a_no_op(models):
    from nerrf_b200 import ingest
    model, scorer = models
    sp = stream.StreamingPlanner(model, scorer)
    assert sp.run(ingest.decode_event_batch(b"")) == [] and not sp.reverted
