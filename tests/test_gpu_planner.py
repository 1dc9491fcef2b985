"""rewards.score and mcts.search CUDA path vs the oracle: BIT-EXACT (needs an H100)."""
import numpy as np
import pytest

from nerrf_b200.ai.planner import mcts, rewards
from nerrf_b200.ai.planner.rewards import Actions
from oracle import mcts_ref as M
from oracle import rewards_ref as RW

pytestmark = pytest.mark.gpu


def _actions(A, seed=2):
    rng = np.random.default_rng(seed)
    p = rng.beta(0.5, 0.5, A).astype(np.float32)
    size = rng.lognormal(np.log(2.0), 1.0, A).astype(np.float32)
    cost = rng.choice([1.0, 10.0, 100.0], A, p=[.9, .09, .01]).astype(np.float32)
    return Actions(p, size, cost)


@pytest.mark.parametrize("A", [1, 31, 100, 1024, 1500, 2048, 4096])
def test_reward_score_bit_exact(A):
    act = _actions(A)
    rng = np.random.default_rng(A)
    applied = rng.random((257, A)) < rng.random((257, 1))
    applied[0] = False; applied[1] = True
    st = rewards.pack_states(applied)
    got = rewards.score(st, act).cpu().numpy()
    want = RW.score(st, act.p, act.size, act.cost)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(st, RW.pack_bits(np.concatenate([applied, np.ones((257, RW.layout(A)[2] - A), bool)], 1)))


def test_bounds_match_oracle():
    for A in (3, 100, 1024):
        act = _actions(A, seed=A)
        root = rewards.empty_state(A); root[0] |= np.uint32(5)
        for rs in (None, root):
            lo, inv = rewards.reward_bounds(act, rs)
            lo2, inv2 = RW.reward_bounds(act.p, act.size, act.cost, rs)
            assert lo == lo2 and inv == inv2
        assert np.array_equal(rewards.empty_state(A), RW.empty_state(A))


CASES = [  # A, R, D, T, seed
    (3, 4, 3, 6, 0),
    (100, 256, 20, 40, 5),
    (40, 64, 10, 30, 1),
    (1024, 4096, 50, 6, 0),          # BASELINE cfg 3 shape (fewer iterations: the numpy oracle is slow)
    (1500, 512, 30, 5, 7),           # NW = 2
    (4096, 1024, 50, 4, 9),          # NW = 4
    (10, 8192, 50, 12, 3),           # R >> A, D > A: rollouts exhaust the action set
    (64, 1, 5, 20, 2),               # R = 1
    (300, 256, 100, 6, 4),           # D > 64: rollouts deeper than the rank-space path (per-step bitset updates), then <= 64 below deeper leaves
    (2048, 512, 64, 5, 6),           # exactly 64 picks: both slot registers of the rank list full; NW = 2
    (90, 128, 64, 10, 8),            # D = 64 with fewer actions than picks after a few levels
]


@pytest.mark.parametrize("A,R,D,T,seed", CASES)
@pytest.mark.parametrize("host_call", [False, True])
def test_mcts_bit_exact(A, R, D, T, seed, host_call):
    act = _actions(A, seed=seed + 10)
    got = mcts.search(act, None, n_rollouts=R, depth=D, seed=seed, iterations=T, host_call=host_call)
    want = M.search(act.p, act.size, act.cost, R=R, D=D, T=T, seed=seed)
    assert np.array_equal(got.root_n, want["root_n"]), "visit counts differ"
    assert np.array_equal(got.root_w.view(np.uint32), want["root_w"].view(np.uint32)), "value sums differ"
    assert got.best == want["best"] and got.num_nodes == want["num_nodes"]


def test_mcts_root_state_and_determinism():
    act = _actions(200, seed=4)
    root = rewards.empty_state(200); root[1] |= np.uint32(0xF0F0)
    a = mcts.search(act, None, 512, 25, 11, iterations=20, root_state=root)
    b = mcts.search(act, None, 512, 25, 11, iterations=20, root_state=root)
    w = M.search(act.p, act.size, act.cost, R=512, D=25, T=20, seed=11, root_state=root)
    assert np.array_equal(a.root_n, b.root_n) and np.array_equal(a.root_w, b.root_w)
    assert np.array_equal(a.root_n, w["root_n"]) and np.array_equal(a.root_w.view(np.uint32), w["root_w"].view(np.uint32))
    assert a.root_n[[36, 37, 38, 39]].sum() == 0


def test_full_size_search_properties():
    """cfg 3 at full size (A=1024, R=4096, D=50, 64 iterations): structural invariants."""
    act = _actions(1024, seed=2)
    T, R = 64, 4096
    r = mcts.search(act, None, R, 50, 0, iterations=T)
    assert r.num_nodes == T                      # one new node per iteration after the first
    assert int(r.root_n.sum()) == R + (T - 1) * R
    assert (r.root_n >= 4).all()                 # stratified first pass touches every action
    q = r.root_q
    assert (q > 0).all() and (q < 1).all()
    gain = (2 * act.p - 1) * act.size - 0.1 * act.cost
    assert (gain > gain[r.best]).sum() < 64      # the recommendation is among the high-gain actions
    # root parallelism: different seeds -> different trees, merged stats add up
    r2 = mcts.search(act, None, R, 50, 1, iterations=T)
    n, w, best = mcts.merge_root_stats([r, r2])
    assert int(n.sum()) == 2 * int(r.root_n.sum()) and not np.array_equal(r.root_w, r2.root_w)


def test_plan_reverts_exactly_the_attacked_files():
    """Semantic check (SURVEY.md 4): with confident scores the plan is the set of encrypted files."""
    rng = np.random.default_rng(0)
    A = 60
    attacked = np.zeros(A, bool); attacked[rng.choice(A, 25, replace=False)] = True
    p = np.where(attacked, 0.95, 0.05).astype(np.float32)
    size = rng.uniform(2, 5, A).astype(np.float32)
    act = Actions(p, size, np.ones(A, np.float32))
    pl = mcts.plan(act, max_steps=40, n_rollouts=1024, depth=40, iterations=8)
    assert sorted(pl.actions) == sorted(np.nonzero(attacked)[0].tolist())
    assert all(b > a for a, b in zip(pl.scores, pl.scores[1:]))


# ---------------------------------------------------------------- planner spec v1: guards (non-separable reward)
def _guarded_actions(A, n_kill, seed):
    rng = np.random.default_rng(seed)
    act = _actions(A, seed)
    size = act.size.copy(); cost = act.cost.copy(); p = act.p.copy()
    size[:n_kill] = 0.0; cost[:n_kill] = 10.0; cost[n_kill:] = 1.0
    guard = rng.integers(-1, n_kill, A).astype(np.int32); guard[:n_kill] = -1; guard[-1] = 0
    return Actions(p, size, cost, guard=guard)


@pytest.mark.parametrize("A,n_kill", [(2, 1), (100, 3), (1024, 32), (1500, 7), (4096, 32)])
def test_guarded_reward_score_bit_exact(A, n_kill):
    act = _guarded_actions(A, n_kill, A)
    rng = np.random.default_rng(A)
    applied = rng.random((129, A)) < rng.random((129, 1))
    st = rewards.pack_states(applied)
    got = rewards.score(st, act).cpu().numpy()
    want = RW.score(st, act.p, act.size, act.cost, act.guard)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    lo, inv = rewards.reward_bounds(act, None)
    lo2, inv2 = RW.reward_bounds(act.p, act.size, act.cost, None, act.guard)
    assert lo == lo2 and inv == inv2


@pytest.mark.parametrize("A,n_kill,R,D,T,seed", [(12, 2, 64, 8, 30, 1), (100, 5, 256, 20, 20, 2), (1024, 32, 4096, 50, 5, 3),
                                                  (1500, 7, 512, 30, 4, 4)])
@pytest.mark.parametrize("host_call", [False, True])
def test_guarded_mcts_bit_exact(A, n_kill, R, D, T, seed, host_call):
    act = _guarded_actions(A, n_kill, seed)
    got = mcts.search(act, None, n_rollouts=R, depth=D, seed=seed, iterations=T, host_call=host_call)
    want = M.search(act.p, act.size, act.cost, R=R, D=D, T=T, seed=seed, guard=act.guard)
    assert np.array_equal(got.root_n, want["root_n"]) and np.array_equal(got.root_w.view(np.uint32), want["root_w"].view(np.uint32))
    assert got.best == want["best"] and got.num_nodes == want["num_nodes"]


def test_search_finds_what_the_threshold_rule_cannot():
    """VERDICT r1 weak #10.  1 kill action + 8 guarded reversions: every single action lowers the reward, so a
    per-action threshold (and a one-step greedy validation) applies nothing; the optimum applies all nine.  The tree
    search must recommend the kill first (its subtree is the only one whose rollouts see the reversions pay off), and
    plan() with a two-move validation horizon must reach the optimum."""
    p = np.array([0.9] * 9, np.float32); size = np.array([0.0] + [1.0] * 8, np.float32)
    cost = np.array([10.0] + [1.0] * 8, np.float32); guard = np.array([-1] + [0] * 8, np.int32)
    act = Actions(p, size, cost, guard=guard)
    st = rewards.pack_states(np.array([[False] * 9, [True] * 9] + [[a == b for b in range(9)] for a in range(9)]))
    sc = rewards.score(st, act).cpu().numpy()
    assert (sc[2:] < sc[0]).all() and sc[1] > sc[0] + 3.0
    r = mcts.search(act, None, n_rollouts=1024, depth=9, seed=0, iterations=32)
    assert r.best == 0, (r.best, r.root_q)
    pl = mcts.plan(act, n_rollouts=1024, depth=9, iterations=32, lookahead=True)
    assert sorted(pl.actions) == list(range(9)) and pl.scores[-1] == pytest.approx(float(sc[1]))


def test_host_session_reuses_buffers():
    act = _actions(1024, seed=2)
    sess = mcts.HostSession(1024, 16, 4096)
    a = mcts.search(act, None, 4096, 50, 0, iterations=16, host_call=sess)
    b = mcts.search(act, None, 4096, 50, 0, iterations=16, host_call=True)
    c = mcts.search(act, None, 4096, 50, 1, iterations=8, host_call=sess)          # smaller search through the same session
    d = mcts.search(act, None, 4096, 50, 1, iterations=8)
    assert np.array_equal(a.root_n, b.root_n) and np.array_equal(a.root_w, b.root_w)
    assert np.array_equal(c.root_n, d.root_n) and np.array_equal(c.root_w, d.root_w)
    sess.close()


@pytest.mark.parametrize("A,cps,guards", [(300, 1, False), (1024, 64, False), (1500, 32, False), (4096, 64, False),
                                          (200, 16, True), (1024, 64, True), (40, 1000, True)])
def test_device_commit_equals_the_host_commit_loop(A, cps, guards):
    """plan(): the validate-and-commit loop as one cooperative launch (nerrf_plan_commit) takes exactly the decisions of the
    host loop over rewards.score calls -- same actions in the same order, same scores bit for bit, same truncation report --
    for separable rewards (spec v0), guarded reversions with tentative lookahead commits (spec v1), NW = 1 / 2 / 4."""
    rng = np.random.default_rng(A + cps)
    act = _actions(A, seed=A)
    if guards:
        k = min(32, max(A // 8, 1))
        guard = np.full(A, -1, np.int32)
        guard[k:] = rng.integers(0, k, A - k)
        cost = act.cost.copy(); cost[:k] = 10.0
        size = act.size.copy(); size[:k] = 0.0
        act = Actions(act.p, size, cost, guard=guard)
    kw = dict(n_rollouts=256, depth=16, iterations=6, commit_per_search=cps, max_steps=min(A, 300), seed=3)
    a = mcts.plan(act, device_commit=True, **kw)
    b = mcts.plan(act, device_commit=False, **kw)
    assert a.actions == b.actions, "committed actions differ"
    assert np.array_equal(np.asarray(a.scores, np.float32).view(np.uint32), np.asarray(b.scores, np.float32).view(np.uint32))
    assert a.truncated == b.truncated and a.remaining_candidates == b.remaining_candidates and len(a.searches) == len(b.searches)
    assert len(a.actions) > 0
