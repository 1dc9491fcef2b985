"""BiLSTM sequence-step attributions on the GPU (DESIGN.md 1.2.1): the input-gradient backward bit for bit against the
training backward, the step kernel bit for bit against its float32 statement and within the gradient tolerance of the
float64 oracle, independence of the batching, the step -> event map of the device sequence builder, and the evidence
carried through the pipeline, the stream (run and live feed), the emitter and the CLI."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from nerrf_b200 import _lib as L, explain as EX, graph as G, ingest, pipeline, stream
from nerrf_b200.ai.models.lstm import LSTMScorer, FEATURE_NAMES
from nerrf_b200.ai.planner import emit
from gpu_util import assert_close_fp32
from seq_explain_ref import dominant_feature, sequence_attributions, step_attr_f32, top_steps

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M1 = os.path.join(ROOT, "tests", "golden", "m1_trace.jsonl")


def batch(B, T, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((B, T, 16)) * 0.7).astype(np.float32)
    ln = rng.integers(0, T + 1, B).astype(np.int32)
    ln[-1] = T
    if B > 1:
        ln[0] = 0
    if B > 2:
        ln[1] = 1; ln[-2] = 1
    return torch.from_numpy(x).cuda(), torch.from_numpy(ln).cuda()


def forward_tape(scorer, x, ln):
    """nerrf_lstm_forward_train -> (hfin, tape, tape_bytes, weights)"""
    B, T, D = x.shape
    w = EX._seq_weights(scorer, x.device)
    wih_t, whh_t, bias = w[0], w[1], w[2]
    tb, wb = C.c_size_t(), C.c_size_t()
    L.check(L.lib().nerrf_lstm_train_workspace_bytes(B, T, D, 256, scorer.num_layers, C.byref(tb), C.byref(wb)), "ws")
    tape = torch.empty(max(tb.value, 16), dtype=torch.uint8, device=x.device)
    hfin = torch.empty(B, 512, device=x.device)
    L.check(L.lib().nerrf_lstm_forward_train(L.ptr(x), L.ptr(ln), B, T, D, 256, scorer.num_layers, L.ptr_array(wih_t),
                                             L.ptr_array(whh_t), L.ptr_array(bias), L.ptr(hfin), L.ptr(tape), tape.numel(),
                                             L.current_stream_ptr()), "forward_train")
    return hfin, tape, wb.value, w


def input_grad(scorer, x, ln, tape, w, ws_bytes=None):
    B, T, D = x.shape
    gb = C.c_size_t()
    L.check(L.lib().nerrf_lstm_input_grad_workspace_bytes(B, T, D, 256, scorer.num_layers, C.byref(gb)), "ig ws")
    n = gb.value if ws_bytes is None else ws_bytes
    ws = torch.empty(max(n, 16), dtype=torch.uint8, device=x.device)
    dseq = torch.full_like(x, float("nan"))
    dhfin = w[5][0].expand(B, 512).contiguous()
    rc = L.lib().nerrf_lstm_input_grad(L.ptr(x), L.ptr(ln), B, T, D, 256, scorer.num_layers, L.ptr_array(w[3]), L.ptr_array(w[4]),
                                       L.ptr(tape), tape.numel(), L.ptr(dhfin), L.ptr(dseq), L.ptr(ws), n, L.current_stream_ptr())
    return rc, dseq


def train_backward(scorer, x, ln, tape, w, ws_bytes):
    B, T, D = x.shape
    dseq = torch.full_like(x, float("nan"))
    dW_ih = [torch.empty_like(a) for a in w[3]]
    dW_hh = [torch.empty_like(a) for a in w[4]]
    db = [torch.empty(1024, device=x.device) for _ in w[3]]
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
    dhfin = w[5][0].expand(B, 512).contiguous()
    L.check(L.lib().nerrf_lstm_backward(L.ptr(x), L.ptr(ln), B, T, D, 256, scorer.num_layers, L.ptr_array(w[3]), L.ptr_array(w[4]),
                                        L.ptr(tape), tape.numel(), L.ptr(dhfin), L.ptr(dseq), L.ptr_array(dW_ih), L.ptr_array(dW_hh),
                                        L.ptr_array(db), L.ptr(ws), ws.numel(), L.current_stream_ptr()), "backward")
    return dseq


@pytest.fixture(scope="module")
def scorer():
    return LSTMScorer(seed=3).cuda()


def bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


# ------------------------------------------------------------------------------------------------------- input grad
@pytest.mark.parametrize("T", [1, 100])
@pytest.mark.parametrize("B", [1, 7, 8, 9, 257, 512])
def test_input_grad_equals_training_backward_bit_for_bit(scorer, B, T):
    x, ln = batch(B, T, B * 100 + T)
    _, tape, ws_train, w = forward_tape(scorer, x, ln)
    tape2 = tape.clone()                                      # the backward consumes the tape: one copy per call
    rc, d1 = input_grad(scorer, x, ln, tape, w)
    assert rc == 0
    d2 = train_backward(scorer, x, ln, tape2, w, ws_train)
    assert np.array_equal(bits(d1), bits(d2))
    valid = (torch.arange(T, device=x.device)[None, :] < ln[:, None].long())
    assert not d1[~valid].any() and torch.isfinite(d1).all()


def test_input_grad_short_workspace(scorer):
    x, ln = batch(9, 20, 5)
    _, tape, _, w = forward_tape(scorer, x, ln)
    gb = C.c_size_t()
    L.check(L.lib().nerrf_lstm_input_grad_workspace_bytes(9, 20, 16, 256, 2, C.byref(gb)), "ws")
    rc, _ = input_grad(scorer, x, ln, tape, w, ws_bytes=gb.value - 1)
    assert rc == -4 and b"workspace too small" in L.lib().nerrf_last_error()


# ---------------------------------------------------------------------------------------------------- explain_steps
def all_steps(x, dseq, ln):
    """every valid step through the kernel (k = T): -> (a [B, T] with NaN at padded steps, feature [B, T])"""
    B, T, _ = x.shape
    st, at, ft, vt = EX.explain_steps(x, dseq, ln, None, T)
    st, at, ft, vt = (a.cpu().numpy() for a in (st, at, ft, vt))
    a = np.full((B, T), np.nan, np.float32); f = np.full((B, T), -2, np.int64)
    for b in range(B):
        m = st[b] >= 0
        assert m.sum() == int(ln[b]) and (st[b, ~m] == -1).all() and (at[b, ~m] == 0).all() and (vt[b] == -1).all()
        a[b, st[b, m]] = at[b, m]; f[b, st[b, m]] = ft[b, m]
    return a, f, st


@pytest.mark.parametrize("B,T", [(16, 100), (9, 1), (33, 37)])
def test_explain_steps_against_float32_statement_and_float64_oracle(scorer, B, T):
    x, ln = batch(B, T, 7 * B + T)
    w = EX._seq_weights(scorer, x.device)
    hfin, dseq = EX.lstm_input_grad_chunk(scorer, w, x, ln)
    xs, ds, lh = x.cpu().numpy(), dseq.cpu().numpy(), ln.cpu().numpy()
    a, f, _ = all_steps(x, dseq, ln)
    want = step_attr_f32(xs, ds)
    fd = dominant_feature(xs, ds)
    z_ref, a_ref = sequence_attributions(scorer.oracle_params(), xs, lh)
    res = EX.explain_sequences(scorer, x, ln, k=8)
    probs = scorer(x, ln)[:, 0].double().cpu().numpy()
    for b in range(B):
        n = int(lh[b])
        assert np.array_equal(a[b, :n].view(np.uint32), want[b, :n].view(np.uint32))     # bit for bit
        assert np.array_equal(f[b, :n], fd[b, :n])
        at_ref = a_ref[b, :n].sum(-1)
        S = np.abs(a_ref[b, :n]).sum(-1)
        rms = float(np.sqrt((at_ref ** 2).mean())) if n else 0.0
        err = np.abs(a[b, :n].astype(np.float64) - at_ref)
        assert (err <= 2e-4 * S + 2e-5 * rms + 1e-30).all(), (b, float(err.max()) if n else 0.0)
        # top-k: the kernel's picks and the oracle's agree outside near-ties at the k-th value
        got = [s["t"] for s in res[b]["steps"]]
        assert len(got) == min(8, n)
        assert got == list(top_steps(a[b], n, 8))                  # the kernel's own ranking of its own a_t
        if got:
            mag = np.abs(at_ref)
            tol = 2 * (2e-4 * S.max() + 2e-5 * rms)
            kth = np.sort(mag)[::-1][len(got) - 1]
            assert all(mag[t] >= kth - tol for t in got)
            assert all(t in got for t in top_steps(at_ref, n, len(got)) if mag[t] > kth + tol)
        z = res[b]["logit"]
        assert abs(z - z_ref[b]) <= 1e-4 * max(1.0, abs(z_ref[b]))
        assert abs(1.0 / (1.0 + np.exp(-z)) - probs[b]) < 1e-5                   # the wgmma inference forward
    sig = torch.sigmoid(torch.tensor([r["logit"] for r in res], dtype=torch.float64))
    assert_close_fp32(sig, torch.from_numpy(probs), rtol=1e-4, atol_rms=1e-5, what="explained logit vs probs")


def test_step_events_and_padding(scorer):
    B, T = 5, 12
    x, ln = batch(B, T, 11)
    ev = torch.arange(B * T, dtype=torch.int64, device=x.device).view(B, T) + 1000
    res = EX.explain_sequences(scorer, x, ln, k=20, step_event=ev)
    for b, r in enumerate(res):
        assert len(r["steps"]) == int(ln[b])
        for s in r["steps"]:
            assert s["event"] == 1000 + b * T + s["t"] and -1 <= s["feature"] < 16
    res = EX.explain_sequences(scorer, x, ln, k=3)
    assert all(s["event"] == -1 for r in res for s in r["steps"])


def test_batching_does_not_change_a_bit(scorer):
    x, ln = batch(40, 100, 21)
    ev = torch.randint(0, 1 << 40, (40, 100), device=x.device)
    base = EX.explain_sequences(scorer, x, ln, k=8, step_event=ev)
    assert json.dumps(base) == json.dumps(EX.explain_sequences(scorer, x, ln, k=8, step_event=ev))        # run to run
    for mb in (1, 7, 512):
        assert json.dumps(EX.explain_sequences(scorer, x, ln, k=8, step_event=ev, max_batch=mb)) == json.dumps(base)
    for i in (0, 1, 17, 39):
        alone = EX.explain_sequences(scorer, x[i:i + 1], ln[i:i + 1], k=8, step_event=ev[i:i + 1])
        assert json.dumps(alone[0]) == json.dumps(base[i])


def test_explain_sequences_refuses_bad_arguments(scorer):
    x, ln = batch(3, 5, 1)
    with pytest.raises(ValueError):
        EX.explain_sequences(scorer, x, ln, k=0)
    with pytest.raises(ValueError):
        EX.explain_sequences(scorer, x, ln, max_batch=0)
    with pytest.raises(ValueError):
        EX.explain_sequences(scorer, x[:, :, :8].contiguous(), ln)
    with pytest.raises(ValueError):
        EX.explain_sequences(scorer, x, ln, step_event=torch.zeros(3, 4, dtype=torch.int64))
    assert EX.explain_sequences(scorer, x[:0], ln[:0]) == []


# ------------------------------------------------------------------------------------------- device sequence builder
def two_source_columns():
    a, _ = stream.fleet_columns(20, 2, seed=3, n_files=12, benign_files=8)
    b, _ = stream.fleet_columns(20, 2, seed=4, n_files=12, benign_files=8)
    return stream.concat_columns([stream.with_source(a, 0), stream.with_source(b, 1)])


@pytest.mark.parametrize("which", ["fleet", "two_sources"])
def test_trace_sequences_ex_events(which):
    cols = stream.fleet_columns(60, 4, seed=2, n_files=20, benign_files=10)[0] if which == "fleet" else two_source_columns()
    ds = stream.DeviceStream(cols, "cuda", observable=True)
    t0, t1 = ds.span()
    for lo, hi in [(t0 - 1, t0 + 40), (t1 - 60, t1)]:
        g = ds.window_graph(lo, hi, 60.0)
        files = np.nonzero(g.meta["node_kind"] == 0)[0]
        pick = np.random.default_rng(0).permutation(files)[:300]
        sq0, ln0 = ds.sequences_device(g, pick)
        sq1, ln1, ev1 = ds.sequences_device(g, pick, events=True)
        assert np.array_equal(bits(sq0), bits(sq1)) and torch.equal(ln0, ln1)
        sq, ln, have, evh = ds.sequences(g, pick, events=True)
        pos = np.searchsorted(have, pick)
        assert np.array_equal(ev1.cpu().numpy(), evh[pos])
        recs = ds.event_records(evh[pos][0, :ln[pos][0]])
        assert all(r["path"] for r in recs)
        if which == "two_sources":
            src = g.meta["node_source"]
            for i in range(0, pick.size, 37):
                rows = evh[pos][i, :ln[pos][i]]
                assert all(r["source"] == src[pick[i]] for r in ds.event_records(rows))


# ------------------------------------------------------------------------------------------------ pipeline / emitter
@pytest.fixture(scope="module")
def toy():
    from nerrf_b200.ai import train as T
    from nerrf_b200.ai.models import GraphSAGE_T
    model, sc = GraphSAGE_T(G.F_IN, 128, 2), LSTMScorer()
    torch.manual_seed(0)
    T.train(model, sc, T.toy_set(range(100, 104)), epochs=25)
    return model.cuda(), sc.cuda()


def test_pipeline_sequence_evidence_keeps_the_plan(toy):
    model, sc = toy
    events = G.read_trace_jsonl(M1)
    g = G.graph_from_events(events, observable=True)
    seq, lengths, nodes, ev = pipeline.file_sequences(events, g, observable=True, return_events=True)
    kw = dict(top_a=64, n_rollouts=256, depth=20, iterations=8, kill_candidates=True)
    r0 = pipeline.run(g, seq, lengths, nodes, model, sc, **kw)
    r1 = pipeline.run(g, seq, lengths, nodes, model, sc, explain_sequences=4, seq_events=ev, **kw)
    assert r0.plan.actions == r1.plan.actions and r0.plan_nodes == r1.plan_nodes
    assert r1.evidence is None and r0.sequence_evidence is None
    kind = np.asarray(g.meta["node_kind"])
    files = {n for n in r1.plan_nodes if kind[n] == 0}
    assert files and set(r1.sequence_evidence) == files
    names, keys = g.meta["names"], g.meta["file_keys"]
    for n, sx in r1.sequence_evidence.items():
        assert 1 <= len(sx["steps"]) <= 4
        for s in sx["steps"]:
            assert keys[G._stem(s["event"]["path"])] == n                           # every event is on that file
    p0, p1 = emit.from_pipeline(g, r0), emit.from_pipeline(g, r1)
    strip = lambda p: [{k: v for k, v in s.items() if not k.startswith("sequence_evidence") and k != "hostile_name"}
                       for s in p["steps"]]
    assert strip(p0) == strip(p1) and emit.to_shell(p0) == emit.to_shell(p1)
    for s in p1["steps"]:
        if s.get("node") in files:
            assert 1 <= len(s["sequence_evidence"]) <= 4 and "sequence_evidence_logit" in s
            assert all(e["feature"] in FEATURE_NAMES or e["feature"] is None for e in s["sequence_evidence"])
        else:
            assert "sequence_evidence" not in s
    # the share of encrypted-file steps whose top sequence event is the ransomware's (reported, not asserted)
    attackers = {int(e["pid"]) for e in events if e["event"] in G.ATTACK_EVENTS}
    lab = np.asarray(g.meta["label"])
    enc = [n for n in files if lab[n] == 1]
    hits = sum(r1.sequence_evidence[n]["steps"][0]["event"]["pid"] in attackers for n in enc)
    print("SEQ_EVIDENCE_RANSOMWARE_TOP_SHARE %d/%d" % (hits, len(enc)))
    # both kinds of evidence: one event_info call
    calls = []
    info = g.meta["event_info"]
    g.meta["event_info"] = lambda ids: (calls.append(len(ids)), info(ids))[1]
    try:
        r2 = pipeline.run(g, seq, lengths, nodes, model, sc, explain=4, explain_sequences=4, seq_events=ev, **kw)
    finally:
        g.meta["event_info"] = info
    assert len(calls) == 1 and r2.plan_nodes == r0.plan_nodes
    assert json.dumps(r2.sequence_evidence, sort_keys=True) == json.dumps(r1.sequence_evidence, sort_keys=True)
    assert set(r2.evidence) == set(r2.plan_nodes)


def test_pipeline_callable_sequences_and_refusals(toy):
    model, sc = toy
    events = G.read_trace_jsonl(M1)
    g = G.graph_from_events(events, observable=True)
    seq, lengths, nodes, ev = pipeline.file_sequences(events, g, observable=True, return_events=True)
    kw = dict(top_a=64, n_rollouts=256, depth=20, iterations=8)
    r1 = pipeline.run(g, seq, lengths, nodes, model, sc, explain_sequences=3, seq_events=ev, **kw)

    def builder(cand, events=False):                           # host builder: the candidates' sequences, sorted by node id
        sel = np.searchsorted(nodes, np.sort(np.asarray(cand)))
        out = (seq[sel], lengths[sel], nodes[sel])
        return out + (ev[sel],) if events else out
    r2 = pipeline.run(g, builder, None, nodes, model, sc, explain_sequences=3, **kw)
    assert r1.plan_nodes == r2.plan_nodes
    assert json.dumps(r1.sequence_evidence, sort_keys=True) == json.dumps(r2.sequence_evidence, sort_keys=True)
    with pytest.raises(NotImplementedError):
        pipeline.run(g, seq, lengths, nodes, model, sc, explain_sequences=2, dist_ctx=pipeline.DistContext(0, 2), **kw)


def _fleet():
    return stream.fleet_columns(30, 2, seed=1, n_files=15, benign_files=10)[0]


def _sp(toy, **kw):
    model, sc = toy
    return stream.StreamingPlanner(model, sc, window_s=60.0, tick_s=30.0, top_a=64, n_rollouts=256, depth=16, iterations=4,
                                   kill_candidates=True, **kw)


def _steps_key(sx, with_syscall=False):
    return [(s["t"], s["attr"], s["feature"], s["event"]["time"], s["event"]["pid"], s["event"]["path"]) for s in sx["steps"]]


def test_stream_sequence_evidence_run_and_live(toy):
    cols = _fleet()
    sp = _sp(toy, explain_sequences=2)
    ticks = sp.run(cols)
    assert any(t.planned for t in ticks)
    for t in ticks:
        assert set(t.sequence_evidence) == set(t.planned)                  # every new file step, and only those
        assert not set(t.sequence_evidence) & sp.killed
        for sx in t.sequence_evidence.values():
            assert 1 <= len(sx["steps"]) <= 2
            assert all(set(s["event"]) >= {"time", "pid", "syscall", "path"} for s in sx["steps"])
    plain = _sp(toy)
    plain.run(cols)
    assert [t.planned for t in plain.ticks] == [t.planned for t in ticks]
    # the live path against run() over the same bytes, delivered in time order (the fleet's events are jittered)
    recs = ingest.encode_columns(cols)
    wire = b"".join(recs[i] for i in np.argsort(cols.timestamp, kind="stable"))
    want = _sp(toy, explain_sequences=2)
    want.run(ingest.decode_event_batch(wire))
    live = _sp(toy, explain_sequences=2)
    fired = []
    for k in range(0, len(wire), 48 << 10):
        fired += live.feed(wire[k:k + (48 << 10)])
    fired += live.flush()
    assert len(fired) == len(want.ticks) and any(t.sequence_evidence for t in fired)
    for a, b in zip(fired, want.ticks):
        assert a.planned == b.planned and set(a.sequence_evidence) == set(b.sequence_evidence)
        for key in b.sequence_evidence:
            assert a.sequence_evidence[key]["logit"] == b.sequence_evidence[key]["logit"]
            assert _steps_key(a.sequence_evidence[key]) == _steps_key(b.sequence_evidence[key])


def test_cli_sequence_evidence(tmp_path):
    from nerrf_b200 import undo
    out = tmp_path / "plan.json"
    undo.main(["--trace", M1, "--train-epochs", "5", "--explain-sequences", "3", "--out", str(out), "--rollouts", "256"])
    plan = json.loads(out.read_text())
    steps = [s for s in plan["steps"] if "node" in s]
    assert steps and all("sequence_evidence" in s and "sequence_evidence_logit" in s for s in steps)
    assert all(1 <= len(s["sequence_evidence"]) <= 3 for s in steps)
    e = steps[0]["sequence_evidence"][0]
    assert set(e) == {"event", "step", "feature", "attribution"} and set(e["event"]) == {"time", "pid", "syscall", "path"}
    out2 = tmp_path / "plan2.json"
    undo.main(["--trace", M1, "--train-epochs", "5", "--explain", "3", "--out", str(out2), "--rollouts", "256"])
    plan2 = json.loads(out2.read_text())
    assert all("evidence" in s and not any(k.startswith("sequence_evidence") for k in s) for s in plan2["steps"] if "node" in s)


def test_cli_two_hosts_carry_host(tmp_path):
    from nerrf_b200 import undo
    a, _ = stream.fleet_columns(12, 2, seed=3, n_files=10, benign_files=6)
    b, _ = stream.fleet_columns(12, 2, seed=4, n_files=10, benign_files=6)
    pa, pb = tmp_path / "a.pb", tmp_path / "b.pb"
    pa.write_bytes(b"".join(ingest.encode_columns(a)))
    pb.write_bytes(b"".join(ingest.encode_columns(b)))
    out = tmp_path / "plan.json"
    undo.main(["--trace", "nodeA=%s" % pa, "--trace", "nodeB=%s" % pb, "--train-epochs", "5", "--explain-sequences", "2",
               "--out", str(out), "--rollouts", "256"])
    plan = json.loads(out.read_text())
    steps = [s for s in plan["steps"] if "sequence_evidence" in s]
    assert steps
    for s in steps:
        assert all(e["event"]["host"] == s["host"] for e in s["sequence_evidence"])
