"""Planner spec v2 on the device: the cover branch of the reward, the search and the commit loop against both oracles,
bit for bit (needs an H100)."""
import numpy as np
import pytest
import torch

from nerrf_b200 import _lib as L
from nerrf_b200.ai.planner import mcts, rewards
from nerrf_b200.ai.planner.rewards import Actions
from oracle import c_restore
from oracle import restore_ref as V2
from oracle import rewards_ref as RW

from test_oracle_restore import MATRIX, instance, states, threshold_instance

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("A,n_restore,guards", MATRIX)
def test_reward_score_ex_bit_exact(A, n_restore, guards):
    p, size, cost, guard, cover = instance(A, n_restore, guards, seed=A + n_restore)
    st = states(A, 300, seed=A)
    act = Actions(p, size, cost, guard=guard, cover=cover)
    got = rewards.score(st, act).cpu().numpy()
    want = V2.score(st, p, size, cost, guard, cover)
    assert np.array_equal(_bits(got), _bits(want))
    assert np.array_equal(_bits(c_restore.score(st, p, size, cost, guard, cover)), _bits(want))


def test_no_cover_unchanged():
    p, size, cost, guard, cover = instance(1500, 8, True, seed=3)
    st = states(1500, 100, seed=4)
    plain = rewards.score(st, Actions(p, size, cost, guard=guard)).cpu().numpy()
    assert np.array_equal(_bits(plain), _bits(RW.score(st, p, size, cost, guard)))
    none = rewards.score(st, Actions(p, size, cost, guard=guard, cover=np.full(1500, -1, np.int32))).cpu().numpy()
    assert np.array_equal(_bits(plain), _bits(none))


def test_abi_rejects_invalid_cover():
    A = 8
    dev = torch.device("cuda")
    p, size, cost = (torch.ones(A, device=dev) for _ in range(3))
    st = torch.from_numpy(RW.empty_state(A).view(np.int32)[None, :].copy()).to(dev)
    out = torch.empty(1, device=dev)
    for cover in ([-1, 0, 1, -1, -1, -1, -1, -1],          # chain: 1 is covered and covers 2
                  [-1, 1, -1, -1, -1, -1, -1, -1],          # covers itself
                  [-1, -1, 9, -1, -1, -1, -1, -1]):         # out of range
        cv = torch.tensor(cover, dtype=torch.int32, device=dev)
        rc = L.lib().nerrf_reward_score_ex(L.ptr(st), 1, L.ptr(p), L.ptr(size), L.ptr(cost), None, L.ptr(cv), A, L.ptr(out),
                                           L.current_stream_ptr())
        assert rc != 0 and b"cover" in L.lib().nerrf_last_error()
    gd = torch.tensor([-1, -1, -1, -1, 0, -1, -1, -1], dtype=torch.int32, device=dev)
    cv = torch.tensor([-1, -1, 0, -1, -1, -1, -1, -1], dtype=torch.int32, device=dev)
    rc = L.lib().nerrf_reward_score_ex(L.ptr(st), 1, L.ptr(p), L.ptr(size), L.ptr(cost), L.ptr(gd), L.ptr(cv), A, L.ptr(out),
                                       L.current_stream_ptr())
    assert rc != 0 and b"guard and a cover" in L.lib().nerrf_last_error()


SEARCH = [  # A, n_restore, R, D, T, seed   (D = 100: the per-step rollout path)
    (60, 3, 128, 50, 12, 1),
    (300, 8, 256, 100, 6, 2),
    (1024, 8, 1024, 50, 6, 3),
    (1500, 8, 512, 50, 4, 4),
    (2048, 16, 256, 100, 3, 5),
    (4096, 8, 256, 50, 3, 6),
    (4096, 31, 256, 100, 3, 7),
]


@pytest.mark.parametrize("A,n_restore,R,D,T,seed", SEARCH)
def test_search_bit_exact(A, n_restore, R, D, T, seed):
    guards = n_restore < 31
    p, size, cost, guard, cover = instance(A, n_restore, guards, seed)
    act = Actions(p, size, cost, guard=guard, cover=cover)
    got = mcts.search(act, None, n_rollouts=R, depth=D, seed=seed, iterations=T)
    want = c_restore.search(p, size, cost, R=R, D=D, T=T, seed=seed, guard=guard, cover=cover)
    assert np.array_equal(got.root_n, want["root_n"]) and np.array_equal(_bits(got.root_w), _bits(want["root_w"]))
    assert got.num_nodes == want["num_nodes"] and (got.lo, got.inv_range) == (float(want["lo"]), float(want["inv_range"]))
    if A <= 300:
        ref = V2.search(p, size, cost, R=R, D=D, T=T, seed=seed, guard=guard, cover=cover)
        assert np.array_equal(ref["root_n"], want["root_n"]) and np.array_equal(_bits(ref["root_w"]), _bits(want["root_w"]))
    host = mcts.search(act, None, n_rollouts=R, depth=D, seed=seed, iterations=T, host_call=True)
    assert np.array_equal(host.root_n, got.root_n) and np.array_equal(_bits(host.root_w), _bits(got.root_w))
    sess = mcts.HostSession(A, T, R)
    try:
        s2 = mcts.search(act, None, n_rollouts=R, depth=D, seed=seed, iterations=T, host_call=sess)
    finally:
        sess.close()
    assert np.array_equal(s2.root_n, got.root_n) and np.array_equal(_bits(s2.root_w), _bits(got.root_w))


@pytest.mark.parametrize("A,n_restore,guards,cps", [(200, 4, True, 1), (1500, 8, True, 16), (300, 8, False, 64)])
def test_plan_device_commit_matches_host_loop(A, n_restore, guards, cps):
    p, size, cost, guard, cover = instance(A, n_restore, guards, seed=A)
    act = Actions(p, size, cost, guard=guard, cover=cover)
    kw = dict(n_rollouts=256, depth=20, iterations=8, commit_per_search=cps, max_steps=40)
    a = mcts.plan(act, device_commit=True, **kw)
    b = mcts.plan(act, device_commit=False, **kw)
    assert a.actions == b.actions and np.array_equal(_bits(a.scores), _bits(b.scores))
    assert len(a.actions) > 0
    # the plan's scores are the exact reward of its prefixes
    applied = np.zeros((len(a.actions) + 1, A), bool)
    for i, x in enumerate(a.actions):
        applied[i + 1:, x] = True
    want = V2.score(rewards.pack_states(applied), p, size, cost, guard, cover)
    assert np.array_equal(_bits(a.scores), _bits(want))


def test_plan_reaches_exhaustive_optimum():
    """18 actions: two directory restores (collateral 0.5 and 6 MB), one kill, 12 files in the first directory (half of
    them guarded by the kill) and 3 guarded files in the second.  The best of all 2^18 subsets is the first restore, the
    kill and the three reversions of the second directory; plan() reaches it."""
    rng = np.random.default_rng(11)
    A = 18
    p = np.concatenate([[0.0, 0.0, 0.95], rng.uniform(0.8, 1.0, 15)]).astype(np.float32)
    size = np.concatenate([[0.5, 6.0, 0.0], rng.uniform(1.0, 3.0, 15)]).astype(np.float32)
    cost = np.array([5.0, 5.0, 10.0] + [1.0] * 15, np.float32)
    cover = np.array([-1, -1, -1] + [0] * 12 + [1] * 3, np.int32)
    guard = np.array([-1, -1, -1] + [2, -1] * 6 + [2] * 3, np.int32)
    act = Actions(p, size, cost, guard=guard, cover=cover)
    st = np.full((1 << A, 32), 0xFFFFFFFF, np.uint32)                 # every subset; padding bits set
    st[:, 0] = np.arange(1 << A, dtype=np.uint32) | np.uint32((0xFFFFFFFF << A) & 0xFFFFFFFF)
    sc = rewards.score(st, act).cpu().numpy()
    assert np.array_equal(_bits(sc[::4099]), _bits(V2.score(st[::4099], p, size, cost, guard, cover)))
    best = int(np.argmax(sc))
    assert [a for a in range(A) if (best >> a) & 1] == [0, 2, 15, 16, 17]
    for dc in (True, False):
        plan = mcts.plan(act, n_rollouts=1024, depth=6, iterations=32, device_commit=dc)
        assert sorted(plan.actions) == [0, 2, 15, 16, 17] and np.float32(plan.scores[-1]) == sc.max()


def test_plan_prefers_the_restore_over_reversions():
    """The threshold-rule counterexample: the plan is the restore alone."""
    p, size, cost, cover = threshold_instance()
    act = Actions(p, size, cost, cover=cover)
    plan = mcts.plan(act, n_rollouts=1024, depth=50, iterations=16)
    assert plan.actions == [0]
    assert int(np.float32(plan.scores[-1]).view(np.uint32)) == 0xC1C7FFFE          # -24.999996, the oracles' value


# ------------------------------------------------------------------------------------------ directory hash on the device
def test_device_dir_hash_equals_host_on_live_streams():
    """nerrf_trace_dir_hash on live window graphs (renames included: merge_renames=False names nodes by the new path) equals
    stream.dir_hash of the node names."""
    from nerrf_b200 import ingest, stream
    from test_gpu_live_stream import _fleet, _records_in_batches, _tracker
    for cols in (_tracker(), _fleet()):
        wire = b"".join(b"".join(b) for b in _records_in_batches(cols))
        for merge in (True, False):
            ds = stream.DeviceStream.live("cuda", observable=True, merge_renames=merge)
            ds.append(wire)
            t0, t1 = ds.span()
            for lo, hi in ((t0 - 1, t1), (t0 + 10, t0 + 70)):
                g = ds.window_graph(lo, hi, 60.0)
                if g is None:
                    continue
                names = g.meta["names"].take(np.arange(g.num_nodes))
                got = g.meta["dir_hash"]().cpu().numpy()
                assert got.tolist() == [stream.dir_hash(n) for n in names]
            ref = stream.DeviceStream(ingest.decode_event_batch(wire), "cuda", observable=True, merge_renames=merge)
            g = ref.window_graph(t0 - 1, t1, 60.0)
            assert torch.equal(g.meta["dir_hash"](), ds.window_graph(t0 - 1, t1, 60.0).meta["dir_hash"]())


# ------------------------------------------------------------------------------------------ end to end: the pipeline
@pytest.fixture(scope="module")
def trained():
    from nerrf_b200.ai import train as T
    from nerrf_b200.ai.models import GraphSAGE_T
    from nerrf_b200.ai.models.lstm import LSTMScorer
    torch.manual_seed(0)
    model, scorer = GraphSAGE_T(32, 128, 2), LSTMScorer()
    T.train(model, scorer, T.toy_set(range(100, 104)), epochs=25, lr=3e-3, device="cuda")
    return model, scorer


def _trace_graph(events):
    from nerrf_b200 import graph as G, pipeline
    g = G.graph_from_events(events, observable=True)
    seq, lengths, nodes = pipeline.file_sequences(events, g, observable=True)
    return g, seq, lengths, nodes


def _fleet_events(n_files, benign_files, n_benign_procs, files_each):
    """lockbit_trace(n_files) in /app/uploads, plus benign processes with their own files in the same directory."""
    from nerrf_b200 import trace_sim
    ev = trace_sim.lockbit_trace(n_files=n_files, benign_files=benign_files, seed=5)
    for k in range(n_benign_procs):
        for e in trace_sim.lockbit_trace(n_files=0, benign_files=files_each, seed=50 + k, pid=2000 + k):
            if e["path"].startswith("/app/uploads/") and "." in e["path"]:
                e["path"] = e["path"].replace("/app/uploads/", "/app/uploads/p%d_" % k)
            ev.append(e)
    from nerrf_b200 import graph as G
    ev.sort(key=lambda e: G._parse_ts(e["timestamp"]))
    return ev


KW = dict(top_a=1000, n_rollouts=1024, depth=40, iterations=8, commit_per_search=64, kill_candidates=True)


def test_lockbit_1000_files_one_restore_and_the_kill(trained):
    from nerrf_b200 import pipeline, trace_sim
    from nerrf_b200.ai.planner import emit
    model, scorer = trained
    ev = trace_sim.lockbit_trace(n_files=1000, benign_files=10, seed=5)
    g, seq, lengths, nodes = _trace_graph(ev)
    names, kind = g.meta["names"], np.asarray(g.meta["node_kind"])
    off = pipeline.run(g, seq, lengths, nodes, model, scorer, **KW)
    default = pipeline.run(g, seq, lengths, nodes, model, scorer, restore_candidates=False, **KW)
    assert off.n_restore == 0 and off.restores == [] and off.actions.cover is None
    assert off.plan.actions == default.plan.actions and off.plan_nodes == default.plan_nodes
    on = pipeline.run(g, seq, lengths, nodes, model, scorer, restore_candidates=True, **KW)
    assert on.n_restore >= 1
    act = on.actions
    up = [i for i in range(on.n_kill, on.n_kill + on.n_restore)
          if act.cover is not None and (act.cover == i).any()
          and all(names[int(on.candidates[j])].startswith("/app/uploads/") for j in np.nonzero(act.cover == i)[0])]
    assert up, "no restore of /app/uploads was proposed"
    r = up[0]
    kills = list(range(on.n_kill))
    # the spec's own arithmetic: {restore, kills} against the plan made without restores
    st = rewards.pack_states([[r] + kills, kills], A=act.A)
    exp_restore = rewards.score(st, act).cpu().numpy()[0]
    assert exp_restore > np.float32(off.plan.scores[-1]), (exp_restore, off.plan.scores[-1])
    # the plan: the restore and the kill, no covered reversion, and a better exact reward than the plan without restores
    assert r in on.plan.actions and [names[n] for n in on.plan_nodes if kind[n] == 1] == ["pid:454"]
    covered = set(int(on.candidates[j]) for j in np.nonzero(act.cover == r)[0])
    assert not covered & set(on.plan_nodes)
    assert [x["dir"] for x in on.restores] == ["/app/uploads"] and set(on.restores[0]["covers"]) == covered
    assert np.float32(on.plan.scores[-1]) > np.float32(off.plan.scores[-1])
    want = V2.score(rewards.pack_states([on.plan.actions], A=act.A), act.p, act.size, act.cost, act.guard, act.cover)
    assert np.float32(on.plan.scores[-1]).view(np.uint32) == want.view(np.uint32)[0]
    # emitted: one restore_snapshot_dir step at the restore's plan position
    plan = emit.from_pipeline(g, on)
    steps = [s for s in plan["steps"] if s["op"] == "restore_snapshot_dir"]
    assert len(steps) == 1 and steps[0]["dir"] == "/app/uploads" and steps[0]["order"] == on.restores[0]["position"]
    assert len(steps[0]["covers"]) == len(covered) and len(steps[0]["validate"]) == len(covered)
    assert ": restore-dir-from-pre-attack-snapshot /app/uploads" in emit.to_shell(plan).splitlines()
    assert "restore_snapshot_dir" not in emit.to_json(emit.from_pipeline(g, off))


def test_fleet_does_not_restore_the_shared_directory(trained):
    from nerrf_b200 import pipeline
    model, scorer = trained
    g, seq, lengths, nodes = _trace_graph(_fleet_events(1000, 10, 3, 300))
    on = pipeline.run(g, seq, lengths, nodes, model, scorer, restore_candidates=True, **KW)
    assert on.n_restore >= 1                                          # proposed: the candidates share /app/uploads ...
    assert on.actions.size[on.n_kill:on.n_kill + on.n_restore].max() > 1000.0   # ... with the other processes' files
    assert on.restores == []                                          # too much collateral: never applied
    names = g.meta["names"]
    assert any(names[n] == "pid:454" for n in on.plan_nodes)


def test_stream_counts_covered_files_as_reverted(trained):
    """The live StreamingPlanner with restore candidates (device-resident stream, device directory hash): the tick that
    sees the whole 1000-file encryption restores /app/uploads, the files it covers count as reverted, and the next tick
    (a later backup job elsewhere; the window still holds the attack) plans none of them again."""
    from datetime import datetime, timedelta
    from nerrf_b200 import ingest, stream, trace_sim
    from test_gpu_live_stream import _records_in_batches
    model, scorer = trained
    ev = trace_sim.lockbit_trace(n_files=1000, benign_files=10, seed=5)
    later = (datetime.fromisoformat(ev[0]["timestamp"]) + timedelta(seconds=2300)).isoformat()
    for e in trace_sim.lockbit_trace(n_files=0, benign_files=20, seed=6, pid=3000, start=later):
        ev.append(dict(e, path=e["path"].replace("/app/uploads", "/srv/backup")))
    cols = ingest.decode_event_batch(ingest.encode_event_batch(ev))
    wire = b"".join(b"".join(b) for b in _records_in_batches(cols))
    sp = stream.StreamingPlanner(model, scorer, window_s=4000.0, tick_s=1750.0, top_a=1000, n_rollouts=1024, depth=40,
                                 iterations=8, kill_candidates=True, restore_candidates=True)
    first = sp.feed(wire)
    assert len(first) == 1 and first[0].restored == ["/app/uploads"] and "pid:454" in sp.killed
    done = set(sp.reverted)
    covered_only = done - set(first[0].planned)
    assert len(covered_only) >= 900 and all(stream.parent_dir(n) == "/app/uploads" for n in covered_only)
    rest = sp.flush()
    assert len(rest) == 1 and not set(rest[0].planned) & done
    assert sp.restored_dirs == [d for t in first + rest for d in t.restored]
