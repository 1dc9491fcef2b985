"""Training on device-built stream windows (needs an H100): per-pair edge labels on the GPU (nerrf_trace_edge_labels)
against the host loader bit for bit, ai.train.stream_examples against the host-built example of the same window, and a
short training run on fleet windows whose checkpoint makes the planner attribute files by the edge head."""
import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G, ingest, pipeline, stream, trace_sim, undo
from nerrf_b200.ai import train as T
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.ai.models.lstm import LSTMScorer

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("lib_built")]


def _lockbit(bystanders, renames=False):
    ev = trace_sim.lockbit_trace(n_files=30, seed=5, benign_files=20, bystanders=bystanders)
    if renames:                             # the encryption as a real rename x.dat -> x.lockbit3 (file <-> file links unmerged)
        for e in ev:
            if e["event"] == "file_encrypt_complete":
                e["new_path"] = e["path"]; e["path"] = e["path"][:-len(".lockbit3")] + ".dat"
    return ingest.decode_event_batch(ingest.encode_event_batch(ev))


def _random_stream():
    """unordered, tied timestamps; every event kind incl. renames and path-less writes"""
    rng = np.random.default_rng(12)
    ev = []
    kinds = ["openat", "write", "rename", "file_encrypt_start", "file_encrypt_complete", "ransom_note_created", "unlink"]
    for _ in range(3000):
        kind = kinds[int(rng.integers(len(kinds)))]
        stem = "/app/uploads/f%d" % rng.integers(150)
        e = {"ts": (1_700_000_000 + int(rng.integers(0, 55)), int(rng.integers(0, 8)) * 125_000_000), "pid": int(rng.integers(1, 6)),
             "syscall": kind, "path": stem + [".dat", ".lockbit3", ""][int(rng.integers(3))], "bytes": int(rng.integers(0, 1 << 22))}
        if kind == "rename":
            e["new_path"] = "/app/uploads/f%d.lockbit3" % rng.integers(150)
        ev.append(e)
    return ingest.decode_event_batch(ingest.encode_event_batch(ev))


def _host_graph(cols, lo, hi, merge, **kw):
    return G.graph_from_events(ingest.events_from_columns(stream.window(cols, lo, hi)), merge_renames=merge, **kw)


def _encryption_times(cols):
    ts = cols.timestamp
    enc = ts[(cols.event_slot == 1) | (cols.event_slot == 2)]
    return float(enc.min()), float(enc.max())


# ------------------------------------------------------------------------------------------------------ 1 edge labels
@pytest.mark.parametrize("trace", ["lockbit0", "lockbit1", "lockbit3", "lockbit1-renames", "random"])
@pytest.mark.parametrize("merge", [True, False])
def test_device_edge_labels_equal_the_host_loader(trace, merge):
    cols = _random_stream() if trace == "random" else _lockbit(int(trace[7]), renames=trace.endswith("renames"))
    ds = stream.DeviceStream(cols, "cuda", observable=True, merge_renames=merge)
    t0, t1 = ds.span()
    if trace == "random":
        windows = [(t0 - 1, t1), (t0 + 10, t0 + 30), (t0 + 40, t1)]
    else:
        e0, e1 = _encryption_times(cols)
        windows = [(t0 - 1, t1),                                 # the whole trace
                   (t0 - 1, e0 - 0.5),                           # before the encryption: no attack event
                   (t0 - 1, 0.5 * (e0 + e1)),                    # cuts the encryption in half
                   (0.5 * (e0 + e1), t1),                        # the second half, and the bystanders after it
                   (e0 + 3.0, e0 + 9.0)]
    seen_attack = seen_quiet = 0
    for lo, hi in windows:
        g = ds.window_graph(lo, hi, 60.0, edge_labels=True)
        want = _host_graph(cols, lo, hi, merge)
        assert np.array_equal(g.rowptr.cpu().numpy(), want.rowptr) and np.array_equal(g.col.cpu().numpy(), want.col)
        lab = g.meta["edge_label"]
        assert lab.is_cuda and lab.dtype == torch.uint8 and lab.shape[0] == g.num_edges
        assert np.array_equal(lab.cpu().numpy(), want.meta["edge_label"]), (lo, hi)
        again = ds.window_graph(lo, hi, 60.0, edge_labels=True).meta["edge_label"]
        assert torch.equal(lab, again)                           # deterministic
        n1 = int(lab.sum())
        seen_attack += n1 > 0
        seen_quiet += n1 == 0
    assert seen_attack and (seen_quiet or trace == "random")
    if trace.startswith("lockbit") and int(trace[7]):
        # with bystanders the edge labels are not the file labels seen from either end
        g = ds.window_graph(t0 - 1, t1, 60.0, edge_labels=True)
        rp = g.rowptr.cpu().numpy().astype(np.int64)
        dst = np.repeat(np.arange(g.num_nodes), np.diff(rp))
        touches = (g.meta["label"][g.col.cpu().numpy()] > 0) | (g.meta["label"][dst] > 0)
        assert (touches & (g.meta["edge_label"].cpu().numpy() == 0)).any()


def test_edge_labels_of_degenerate_graphs():
    c = lambda a: torch.from_numpy(np.asarray(a)).cuda()
    i32, u8 = np.int32, np.uint8
    # E = 0
    out = G.edge_labels_device(c(np.array([0], i32)), c(np.array([1], i32)), c(np.array([1], u8)),
                               c(np.zeros(4, i32)), c(np.zeros(0, i32)), 3)
    assert out.shape == (0,) and out.dtype == torch.uint8
    # no event: nothing is an attack pair
    rp, col = np.array([0, 1, 2], i32), np.array([1, 0], i32)
    out = G.edge_labels_device(c(np.zeros(0, i32)), c(np.zeros(0, i32)), c(np.zeros(0, u8)), c(rp), c(col), 2)
    assert out.tolist() == [0, 0]
    # one attack event 0 -> 1; a non-attack event 2 -> 1; an int64 rowptr; ids outside [0, N) match nothing
    P, F, S = np.array([0, 2, 5], i32), np.array([1, 1, 1], i32), np.array([2, 4, 3], u8)
    rp = np.array([0, 1, 3, 4], np.int64); col = np.array([1, 0, 2, 1], i32)       # rows: 0 <- 1, 1 <- 0, 1 <- 2, 2 <- 1
    out = G.edge_labels_device(c(P), c(F), c(S), c(rp), c(col), 3)
    assert out.tolist() == [1, 1, 0, 0]


# ------------------------------------------------------------------------------------------------- 2 stream examples
def test_edge_labels_off_leaves_the_window_graph_unchanged():
    cols, _ = stream.fleet_columns(40, 4, seed=3, bystanders=2)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    for lo, hi in [(t0 + 10, t0 + 70), (t0 + 40, t1)]:
        a, b = ds.window_graph(lo, hi, 60.0), ds.window_graph(lo, hi, 60.0, edge_labels=True)
        assert "edge_label" not in a.meta and b.meta["edge_label"].shape[0] == a.num_edges
        for k in ("rowptr", "col", "ew", "x"):
            assert torch.equal(getattr(a, k), getattr(b, k)), k
        for k in ("label", "node_kind", "size_mb"):
            assert np.array_equal(a.meta[k], b.meta[k]), k
        assert torch.equal(a.meta["name_hash"], b.meta["name_hash"]) and torch.equal(a.meta["perm"], b.meta["perm"])


def test_stream_examples_equal_the_host_built_window():
    cols, _ = stream.fleet_columns(40, 4, seed=3, bystanders=2)
    exs = T.stream_examples(cols, 4, window_s=60.0, seed=1, files_per_window=64)
    assert len(exs) == 4
    for ex in exs:
        lo, hi = ex["window"]
        ev = ingest.events_from_columns(stream.window(cols, lo, hi))
        want = G.graph_from_events(ev, observable=True, window=60.0)
        assert np.array_equal(ex["rowptr"].cpu().numpy(), want.rowptr) and np.array_equal(ex["col"].cpu().numpy(), want.col)
        assert np.array_equal(ex["label"].cpu().numpy(), want.meta["label"].astype(np.float32))
        assert np.array_equal(ex["is_file"].cpu().numpy(), want.meta["node_kind"] == 0)
        assert np.array_equal(ex["edge_label"].cpu().numpy(), want.meta["edge_label"])
        assert np.allclose(ex["x"].cpu().numpy(), want.x, rtol=1e-6, atol=1e-7)
        assert np.allclose(ex["ew"].cpu().numpy(), want.ew, rtol=1e-6, atol=0)
        seq, lengths, nodes = pipeline.file_sequences(ev, want, observable=True)
        pick = np.searchsorted(nodes, ex["seq_nodes"])
        assert np.array_equal(nodes[pick], ex["seq_nodes"])
        assert np.array_equal(ex["lengths"].cpu().numpy(), lengths[pick])
        assert np.allclose(ex["seq"].cpu().numpy(), seq[pick], rtol=1e-6, atol=1e-7)
        assert np.array_equal(ex["seq_label"].cpu().numpy(), want.meta["label"][ex["seq_nodes"]].astype(np.float32))
        # the file sample is class balanced as far as the window allows
        y = want.meta["label"][ex["seq_nodes"]]
        n_pos = int((want.meta["label"][want.meta["node_kind"] == 0] > 0).sum())
        assert int(y.sum()) == min(n_pos, 32) and len(y) <= 64
        assert ex["events"] is None
    assert any(float(ex["label"].sum()) > 0 for ex in exs)


# -------------------------------------------------------------------------------------------------- 3 training gate
def test_training_on_fleet_windows_meets_the_gates(tmp_path):
    torch.manual_seed(0)
    train_set = T.stream_examples(stream.fleet_columns(40, 4, seed=0, bystanders=2)[0], 8, seed=0, files_per_window=256)
    cols, enc, bad = stream.fleet_columns(40, 4, seed=1, bystanders=2, return_pids=True)
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    test_set = T.stream_examples(ds, 4, seed=1, files_per_window=256)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, train_set, epochs=40, lr=3e-3, device="cuda", lstm_backward="library", edge_weight=1.0)
    auc = T.evaluate(model, scorer, test_set, device="cuda", edges=True)
    assert auc["gnn_auc"] >= 0.90 and auc["edge_auc_encrypted"] >= 0.90, auc
    path = tmp_path / "w.pt"
    torch.save({"sage": model.state_dict(), "lstm": scorer.state_dict(), "layers": 2, "edge_head_trained": True}, path)
    m2, s2 = undo.load_models(str(path), 0)
    assert m2.edge_head_trained is True
    m2.cuda(); s2.cuda()
    t0, t1 = ds.span()
    g = ds.window_graph(t1 - 60.0, t1, 60.0)
    nodes = np.nonzero(g.meta["node_kind"] == 0)[0]
    res = pipeline.run(g, lambda cand: (*ds.sequences_device(g, cand), None), None, nodes, m2, s2, top_a=1024,
                       n_rollouts=512, depth=24, iterations=8, commit_per_search=32, kill_candidates=True)
    assert res.kill_attribution == "edges"
    names = g.meta["names"]
    killed = {nm for v, nm in zip(res.plan_nodes, names.take(res.plan_nodes)) if g.meta["node_kind"][int(v)] == 1}
    assert killed and killed <= bad
