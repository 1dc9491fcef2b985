"""BiLSTM sequence-step attributions without a GPU (DESIGN.md 1.2.1): the float64 oracle against central differences,
the valid-step and ranking rules, the event of every sequence step on the host builders, the plan fields, and the
argument checks of the new C-ABI entry points."""
import ctypes
import json
import os

import numpy as np
import pytest

from nerrf_b200 import graph as G, ingest, pipeline
from nerrf_b200.ai.models.lstm import FEATURE_NAMES, D_IN
from nerrf_b200.ai.planner import emit
from oracle import lstm_bwd_ref as LB, lstm_ref as LR
from seq_explain_ref import dominant_feature, sequence_attributions, step_attr_f32, top_steps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M1 = os.path.join(ROOT, "tests", "golden", "m1_trace.jsonl")


def small(seed=0, B=3, T=6, hidden=8):
    params = LR.make_params(in_dim=D_IN, hidden=hidden, num_layers=2, seed=seed)
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, T, D_IN))
    return params, x


def test_oracle_matches_central_differences():
    params, x = small(B=3, T=6)
    ln = np.array([6, 3, 1])
    z, a = sequence_attributions(params, x, ln)
    assert np.allclose(z, LB.logits(params, x, ln)[:, 0], rtol=0, atol=1e-12)
    eps = 1e-6
    rng = np.random.default_rng(1)
    for b in range(3):
        for _ in range(12):
            t, d = int(rng.integers(0, ln[b])), int(rng.integers(0, D_IN))
            up, dn = x.copy(), x.copy()
            up[b, t, d] += eps; dn[b, t, d] -= eps
            g = (LB.logits(params, up, ln)[b, 0] - LB.logits(params, dn, ln)[b, 0]) / (2 * eps)
            assert abs(x[b, t, d] * g - a[b, t, d]) <= 1e-7 * max(1.0, abs(a[b, t, d])), (b, t, d)


def test_padded_steps_change_nothing_and_a_len1_sequence_has_one_step():
    params, x = small(B=2, T=7, seed=2)
    ln = np.array([4, 1])
    z, a = sequence_attributions(params, x, ln)
    y = x.copy()
    y[0, 4:] = 123.0; y[1, 1:] = -7.0
    z2, a2 = sequence_attributions(params, y, ln)
    assert np.array_equal(z, z2) and np.array_equal(a, a2)
    assert not a[0, 4:].any() and not a[1, 1:].any()
    a_t = a.sum(-1)
    assert list(top_steps(a_t[1], 1, 8)) == [0]
    assert a[1, 0].any()


def test_ranking_and_dominant_feature_rules():
    a = np.array([1.0, -1.0, 0.5, np.nan, -2.0, 1.0], np.float32)
    assert list(top_steps(a, 6, 6)) == [4, 0, 1, 5, 2, 3]           # |a| descending, ties to the lower t, NaN last
    assert list(top_steps(a, 3, 8)) == [0, 1, 2]                    # only the valid steps
    x = np.array([[1.0, 2.0, -2.0, 0.0], [0.0, 0.0, 0.0, 0.0]], np.float32)
    g = np.array([[1.0, 1.0, 1.0, 5.0], [1.0, 2.0, 3.0, 4.0]], np.float32)
    assert list(dominant_feature(x, g)) == [1, -1]                  # |2| == |-2|: the lower d; all-zero terms: -1
    p = np.float32([0.1, 0.2, 0.3]) * np.float32([3.0, 3.0, 3.0])
    want = (p[0] + p[1]) + p[2]
    assert step_attr_f32(np.float32([[0.1, 0.2, 0.3]]), np.float32([[3.0, 3.0, 3.0]]))[0] == want


def _check_steps(ev, ln, nodes, t_max, node_of, time_of, all_of):
    """every valid step's event is on its file, in time order, and they are the file's last t_max events"""
    for i, f in enumerate(nodes.tolist()):
        e = ev[i, :ln[i]]
        assert (e >= 0).all() and (ev[i, ln[i]:] == -1).all()
        assert all(node_of(j) == f for j in e.tolist())
        ts = [time_of(j) for j in e.tolist()]
        assert ts == sorted(ts)
        mine = all_of(f)
        assert ln[i] == min(len(mine), t_max) and list(e) == mine[-ln[i]:]


@pytest.mark.parametrize("t_max", [4, 100])
def test_file_sequences_events(t_max):
    events = G.read_trace_jsonl(M1)
    g = G.graph_from_events(events, observable=True)
    seq0, ln0, nodes0 = pipeline.file_sequences(events, g, t_max=t_max, observable=True)
    seq, ln, nodes, ev = pipeline.file_sequences(events, g, t_max=t_max, observable=True, return_events=True)
    assert np.array_equal(seq, seq0) and np.array_equal(ln, ln0) and np.array_equal(nodes, nodes0)
    assert ev.shape == (nodes.size, t_max) and ev.dtype == np.int64
    evs = G.resolve_event_paths(events)
    keys = g.meta["file_keys"]
    node_of = lambda j: keys.get(G._stem(evs[j]["path"]))
    by = {}
    for j in range(len(evs)):
        by.setdefault(node_of(j), []).append(j)
    _check_steps(ev, ln, nodes, t_max, node_of, lambda j: G._parse_ts(evs[j]["timestamp"]), lambda f: by[f])
    ids = np.unique(ev[ev >= 0])
    recs = dict(zip(ids.tolist(), g.meta["event_info"](ids)))
    names = g.meta["names"]
    for i, f in enumerate(nodes.tolist()):
        for j in ev[i, :ln[i]].tolist():
            assert G._stem(recs[j]["path"]) == G._stem(names[f])


@pytest.mark.parametrize("t_max", [4, 100])
def test_sequences_from_columns_events(t_max):
    events = G.read_trace_jsonl(M1)
    cols = ingest.resolve_columns(ingest.decode_event_batch(ingest.encode_event_batch(events)))
    seq0, ln0, nodes0 = ingest.sequences_from_columns(cols, t_max=t_max, observable=True)
    seq, ln, nodes, ev = ingest.sequences_from_columns(cols, t_max=t_max, observable=True, return_events=True)
    assert np.array_equal(seq, seq0) and np.array_equal(ln, ln0) and np.array_equal(nodes, nodes0)
    order = np.argsort(cols.timestamp, kind="stable")
    _, node_f, _, _, _, _ = ingest.intern_nodes(cols, order, True)
    by = {}
    for r in order.tolist():
        by.setdefault(int(node_f[r]), []).append(r)
    _check_steps(ev, ln, nodes, t_max, lambda r: int(node_f[r]), lambda r: float(cols.timestamp[r]), lambda f: by[f])
    # the same steps as the per-event builder: a row is order[index into the time-sorted events]
    evl = ingest.events_from_columns(cols)
    gh = G.graph_from_events(evl, observable=True)
    _, _, nodes_h, ev_h = pipeline.file_sequences(evl, gh, t_max=t_max, observable=True, return_events=True)
    assert np.array_equal(nodes_h, nodes)
    assert np.array_equal(ev, np.where(ev_h >= 0, order[np.maximum(ev_h, 0)], -1))
    # only_nodes keeps each kept file's events
    pick = nodes[::3]
    _, _, nodes_s, ev_s = ingest.sequences_from_columns(cols, t_max=t_max, observable=True, only_nodes=pick, return_events=True)
    assert np.array_equal(nodes_s, pick) and np.array_equal(ev_s, ev[::3])
    recs = ingest.column_event_records(cols, ev[0, :ln[0]])
    assert all(r["path"] for r in recs)


# ----------------------------------------------------------------------------------------------------------- emitter
def _seq_ex(path="/data/a.dat", pid=7, logit=2.5):
    return {"logit": logit, "steps": [
        {"t": 3, "attr": 0.75, "feature": 1, "event": {"time": 1.5, "pid": pid, "syscall": "write", "path": path}},
        {"t": 0, "attr": -0.25, "feature": -1, "event": None}]}


def test_emitter_sequence_fields_and_unchanged_plans():
    names = ["pid:7", "/data/a.dat.lockbit3", "/data/b.txt"]
    base = dict(scores=[-3.0, -2.0, -1.0], size_mb=np.ones(3, np.float32), node_score=np.full(3, 0.5, np.float32))
    p0 = emit.undo_plan(names, [0, 1, 2], **base)
    p1 = emit.undo_plan(names, [0, 1, 2], sequence_evidence=None, **base)
    assert emit.to_json(p0) == emit.to_json(p1)
    p2 = emit.undo_plan(names, [0, 1, 2], sequence_evidence={1: _seq_ex(), 2: _seq_ex("/data/b.txt", logit=-1.0)}, **base)
    s = {st["node"]: st for st in p2["steps"]}
    assert "sequence_evidence" not in s[0]                           # a kill carries none
    se = s[1]["sequence_evidence"]
    assert se[0] == {"event": {"time": 1.5, "pid": 7, "syscall": "write", "path": "/data/a.dat"}, "step": 3,
                     "feature": FEATURE_NAMES[1], "attribution": 0.75}
    assert se[1]["event"] is None and se[1]["feature"] is None
    assert s[1]["sequence_evidence_logit"] == 2.5 and s[2]["sequence_evidence_logit"] == -1.0
    assert "hostile_name" not in s[1]
    strip = lambda p: [{k: v for k, v in st.items() if not k.startswith("sequence_evidence")} for st in p["steps"]]
    assert strip(p2) == strip(p0)
    assert emit.to_shell(p2) == emit.to_shell(p0)
    json.loads(emit.to_json(p2))


def test_emitter_hostile_event_path_and_hosts():
    names = ["/data/a.dat.lockbit3"]
    p = emit.undo_plan(names, [0], sequence_evidence={0: _seq_ex("/data/a\n; rm -rf /")})
    assert p["steps"][0]["hostile_name"] is True
    assert "rm -rf" not in emit.to_shell(p)
    ex = _seq_ex()
    ex["steps"][0]["event"]["source"] = 1
    p = emit.undo_plan(names, [0], sequence_evidence={0: ex}, host_names=["h0", "h1"])
    assert p["steps"][0]["sequence_evidence"][0]["event"]["host"] == "h1"
    with pytest.raises(ValueError):
        emit.undo_plan(names, [0], sequence_evidence={0: ex}, host_names=["h0", "bad host"])


def test_from_pipeline_without_the_option_is_unchanged():
    class R:
        node_score = np.full(2, 0.5, np.float32)
        plan_nodes = [1]
        plan = type("P", (), {"scores": [-2.0, -1.0], "truncated": False, "remaining_candidates": 0})()
        restores = []
        evidence = None
    g = G.TemporalGraph(None, None, None, None, {"names": ["pid:1", "/x.lockbit3"], "size_mb": np.ones(2, np.float32)})
    a = emit.from_pipeline(g, R())
    r = R(); r.sequence_evidence = None
    assert emit.to_json(emit.from_pipeline(g, r)) == emit.to_json(a)
    r.sequence_evidence = {1: _seq_ex()}
    b = emit.from_pipeline(g, r)
    assert b["steps"][0]["sequence_evidence_logit"] == 2.5


# ------------------------------------------------------------------------------------ argument errors of the C ABI
def _fake(n):
    return ctypes.c_void_p(n << 20)


def _ptrs(n, base):
    arr = (ctypes.c_void_p * n)()
    for i in range(n):
        arr[i] = (base + i) << 20
    return arr


def test_new_entry_points_refuse_bad_arguments(lib_built):
    from nerrf_b200 import _lib
    h = _lib.lib()
    wb, tb, tw = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    assert h.nerrf_lstm_input_grad_workspace_bytes(4, 100, 16, 128, 2, ctypes.byref(wb)) == -1      # H != 256
    assert h.nerrf_lstm_input_grad_workspace_bytes(4, 100, 16, 256, 2, None) == -1
    assert h.nerrf_lstm_input_grad_workspace_bytes(4, 100, 16, 256, 2, ctypes.byref(wb)) == 0
    assert wb.value == 4 * 100 * 2 * 256 * 4                          # the dout buffer only
    assert h.nerrf_lstm_train_workspace_bytes(4, 100, 16, 256, 2, ctypes.byref(tb), ctypes.byref(tw)) == 0
    assert tw.value > wb.value                                         # the training call adds the weight-gradient partials
    W = lambda: _ptrs(4, 40)

    def ig(H=256, dseq=_fake(12), dhfin=_fake(10), tape_bytes=tb.value, ws_bytes=wb.value, ws=_fake(11)):
        return h.nerrf_lstm_input_grad(_fake(1), _fake(2), 4, 100, 16, H, 2, W(), W(), _fake(9), tape_bytes, dhfin, dseq,
                                       ws, ws_bytes, None)
    assert ig(H=512) == -1 and b"H == 256" in h.nerrf_last_error()
    assert ig(dseq=None) == -1 and b"null" in h.nerrf_last_error()
    assert ig(dhfin=None) == -1
    assert ig(ws=ctypes.c_void_p((11 << 20) + 4)) == -1 and b"aligned" in h.nerrf_last_error()
    assert ig(tape_bytes=tb.value - 1) == -4 and b"tape too small" in h.nerrf_last_error()
    assert ig(ws_bytes=wb.value - 1) == -4 and b"workspace too small" in h.nerrf_last_error()
    assert h.nerrf_lstm_input_grad(None, None, 0, 100, 16, 256, 2, None, None, None, 0, None, None, None, 0, None) == 0

    def st(B=4, T=100, D=16, k=8, seq=_fake(1), out=_fake(5)):
        return h.nerrf_lstm_explain_steps(seq, _fake(2), _fake(3), B, T, D, None, k, out, _fake(6), _fake(7), _fake(8), None)
    assert st(k=0) == -1 and b"k must" in h.nerrf_last_error()
    assert st(k=1025) == -1
    assert st(D=0) == -1 and st(D=1025) == -1 and st(T=0) == -1 and st(B=-1) == -1
    assert st(seq=None) == -1 and b"null" in h.nerrf_last_error()
    assert st(out=None) == -1
    assert st(B=0, seq=None, out=None) == 0

    def ts(n=4, t_max=100, seq=_fake(6)):
        return h.nerrf_trace_sequences_ex(_fake(1), n, _fake(2), 0, _fake(3), _fake(4), _fake(5), _fake(7), _fake(8), _fake(9),
                                          0.0, 1.0, t_max, seq, _fake(10), None, None)
    assert ts(t_max=0) == -1 and ts(n=-1) == -1
    assert ts(seq=None) == -1 and b"null" in h.nerrf_last_error()
    assert ts(n=0) == 0
