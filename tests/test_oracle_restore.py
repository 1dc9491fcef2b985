"""Planner spec v2 (cover / "restore from backup" actions): the numpy oracle against the C oracle, bit for bit, and the
properties the planner relies on.  CPU only."""
import itertools

import numpy as np
import pytest

from oracle import c_oracle, c_restore
from oracle import mcts_ref as M
from oracle import restore_ref as V2
from oracle import rewards_ref as RW


def instance(A, n_restore, guards, seed):
    """Random actions with `n_restore` restore actions in slots 0.. (after the kills when guards are on) covering random
    actions, and optionally kill actions guarding others."""
    rng = np.random.default_rng(seed)
    p = rng.beta(0.5, 0.5, A).astype(np.float32)
    size = rng.lognormal(np.log(2.0), 1.0, A).astype(np.float32)
    cost = rng.choice([1.0, 10.0, 100.0], A, p=[.9, .09, .01]).astype(np.float32)
    n_kill = min(4, 32 - n_restore, A - n_restore - 1) if guards else 0
    kills = np.arange(n_kill)
    restores = np.arange(n_kill, n_kill + n_restore)
    cost[kills] = 10.0; cost[restores] = 100.0; p[restores] = 0.0
    guard = None
    if guards:
        guard = np.full(A, -1, np.int32)
        sel = rng.random(A) < 0.5
        sel[:n_kill + n_restore] = False
        guard[sel] = rng.choice(kills, sel.sum())
    cover = np.full(A, -1, np.int32)
    sel = rng.random(A) < 0.7
    sel[:n_kill + n_restore] = False
    cover[sel] = rng.choice(restores, sel.sum())
    return p, size, cost, guard, cover


def states(A, B, seed):
    rng = np.random.default_rng(seed)
    _, _, A_pad, _ = RW.layout(A)
    bits = np.ones((B, A_pad), bool)
    bits[:, :A] = rng.random((B, A)) < rng.random((B, 1))
    bits[0, :A] = False
    bits[1, :A] = True
    mixed = bits[2:10]                                              # word 0 (kills / restores) mixed
    mixed[:, :32] = rng.random((mixed.shape[0], 32)) < 0.5
    return RW.pack_bits(bits)


MATRIX = [(A, nr, g) for A in (40, 1024, 1500, 4096) for nr in (1, 8, 31) for g in (False, True)
          if not (g and nr == 31)]


@pytest.mark.parametrize("A,n_restore,guards", MATRIX)
def test_numpy_and_c_oracles_agree(A, n_restore, guards):
    p, size, cost, guard, cover = instance(A, n_restore, guards, seed=A + n_restore)
    st = states(A, 64, seed=A)
    a = V2.score(st, p, size, cost, guard, cover)
    b = c_restore.score(st, p, size, cost, guard, cover)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("A", [5, 100, 1024, 2048, 4096])
def test_no_cover_is_spec_v1(A):
    p, size, cost, guard, _ = instance(A, 1, A > 10, seed=A)
    st = states(A, 32, seed=A + 1)
    want = RW.score(st, p, size, cost, guard)
    for cover in (None, np.full(A, -1, np.int32)):
        for got in (V2.score(st, p, size, cost, guard, cover), c_restore.score(st, p, size, cost, guard, cover)):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert np.array_equal(c_oracle.score(st, p, size, cost, guard).view(np.uint32), want.view(np.uint32))
    assert V2.reward_bounds(p, size, cost, None, guard, None) == RW.reward_bounds(p, size, cost, None, guard)


def test_known_answers():
    """A = 4: action 0 restores the directory of actions 2 and 3; action 1 kills the writer of action 3."""
    p = np.array([0.0, 0.5, 0.5, 0.5], np.float32)
    size = np.array([3.0, 0.0, 2.0, 4.0], np.float32)
    cost = np.array([100.0, 10.0, 1.0, 1.0], np.float32)
    guard = np.array([-1, -1, -1, 1], np.int32)
    cover = np.array([-1, -1, 0, 0], np.int32)
    # u = (0, 0, 1, 2), v = (3, 0, 1, 2), vw_3 = 2 + 0.5 * 2 = 3
    want = {(): -(0 + 0 + 1 + 2),
            (0,): -((3 + 1 + 3) + 10.0),            # restore: 2 and 3 restored; 3's writer alive -> vw
            (0, 1): -((3 + 1 + 2) + 11.0),          # + kill: 3 sticks
            (2,): -((1 + 2) + 0.1),                 # one reversion
            (0, 2): -((3 + 1 + 3) + 10.1),          # a covered reversion only adds its downtime
            (1, 3): -((1 + 2) + 1.1)}
    for applied, w in want.items():
        st = RW.pack_bits(np.concatenate([np.isin(np.arange(4), applied), np.ones(1020, bool)])[None, :])
        for got in (V2.score(st, p, size, cost, guard, cover), c_restore.score(st, p, size, cost, guard, cover)):
            assert got[0] == np.float32(w), (applied, got[0], w)


def _exhaustive(A, p, size, cost, guard, cover):
    bits = np.ones((1 << A, 1024), bool)
    bits[:, :A] = (np.arange(1 << A)[:, None] >> np.arange(A)) & 1
    return RW.pack_bits(bits)


@pytest.mark.parametrize("seed", range(6))
def test_bounds_contain_every_score(seed):
    rng = np.random.default_rng(seed)
    A = 10
    p, size, cost, guard, cover = instance(A, 2, seed % 2 == 1, seed)
    st = _exhaustive(A, p, size, cost, guard, cover)
    sc = V2.score(st, p, size, cost, guard, cover)
    lo, inv = V2.reward_bounds(p, size, cost, None, guard, cover)
    hi = float(lo) + 1.0 / float(inv)
    assert sc.min() >= lo - 1e-4 and sc.max() <= hi + 1e-4
    # random roots of a large instance: every superset sampled stays inside the bounds
    p, size, cost, guard, cover = instance(1500, 8, True, seed)
    root = states(1500, 4, seed)[3]
    lo, inv = V2.reward_bounds(p, size, cost, root, guard, cover)
    hi = float(lo) + 1.0 / float(inv)
    sup = states(1500, 200, seed + 7) | root[None, :]
    sc = V2.score(sup, p, size, cost, guard, cover)
    assert sc.min() >= lo - 1e-2 and sc.max() <= hi + 1e-2
    assert not np.array_equal(V2.reward_bounds(p, size, cost, None, guard, cover), V2.reward_bounds(p, size, cost, None, guard))


def test_validation():
    A = 6
    p = np.full(A, 0.5, np.float32); s = np.ones(A, np.float32); c = np.ones(A, np.float32)
    bad = [([-2, -1, -1, -1, -1, -1], None),       # below -1
           ([-1, -1, 6, -1, -1, -1], None),        # >= A
           ([-1, 1, -1, -1, -1, -1], None),        # covers itself
           ([-1, 0, 1, -1, -1, -1], None),         # 1 is covered by 0 and covers 2: a chain
           ([-1, -1, 0, 0, -1, -1], [-1, -1, -1, -1, 0, -1])]  # 0 is a cover and a guard target
    for cover, guard in bad:
        with pytest.raises(ValueError):
            V2.score(RW.empty_state(A)[None, :], p, s, c, guard, np.array(cover, np.int32))
    with pytest.raises(ValueError):
        V2.check_cover(np.full(40, -1, np.int32) + np.eye(40, dtype=np.int32)[39] * 33, None, 40)   # target >= 32
    from nerrf_b200.ai.planner.rewards import Actions
    for cover, guard in bad:
        with pytest.raises(ValueError):
            Actions(p, s, c, guard=None if guard is None else np.array(guard, np.int32), cover=np.array(cover, np.int32))
    assert Actions(p, s, c, cover=np.full(A, -1, np.int32)).cover is None


def threshold_instance():
    """150 files (p = 0.9, size 1, cost 1) in one directory and the restore of that directory (collateral 0)."""
    A = 151
    p = np.array([0.0] + [0.9] * 150, np.float32)
    size = np.array([0.0] + [1.0] * 150, np.float32)
    cost = np.array([100.0] + [1.0] * 150, np.float32)
    cover = np.array([-1] + [0] * 150, np.int32)
    return p, size, cost, cover


def test_threshold_rule_is_provably_wrong_under_spec_v2():
    """Every action alone improves the empty state, so a threshold rule applies all of them (-40); the restore alone
    scores -25, every reversion added to it only adds 0.1 of downtime, and the reversions without it score -30."""
    p, size, cost, cover = threshold_instance()
    A = 151

    def sc(applied):
        bits = np.ones((1, 1024), bool)
        bits[0, :A] = np.isin(np.arange(A), list(applied))
        st = RW.pack_bits(bits)
        a = V2.score(st, p, size, cost, None, cover)[0]
        assert a.view(np.uint32) == c_restore.score(st, p, size, cost, None, cover)[0].view(np.uint32)
        return a

    empty = sc([])
    singles = np.array([sc([a]) for a in range(A)])
    assert (singles > empty).all()
    everything, restore, reverts = sc(range(A)), sc([0]), sc(range(1, A))
    # the oracles' exact fp32 results (0.1 and 0.9 are not exact in fp32)
    bits = lambda x: int(np.float32(x).view(np.uint32))
    assert bits(empty) == 0xC306FFFD                                 # -134.99995
    assert bits(restore) == 0xC1C7FFFE                               # -24.999996
    assert bits(everything) == 0xC21FFFFF                            # -39.999996
    assert bits(reverts) == 0xC1EFFFFE                               # -29.999996
    assert restore > reverts > everything
    for k in (1, 2, 50):                                           # any extra reversion only adds downtime
        assert sc([0] + list(range(1, 1 + k))) < restore


@pytest.mark.parametrize("A,R,D,T,guards,seed", [(40, 64, 10, 12, True, 1), (100, 128, 20, 8, False, 2), (60, 32, 80, 5, True, 3)])
def test_search_oracles_agree(A, R, D, T, guards, seed):
    p, size, cost, guard, cover = instance(A, 3, guards, seed)
    a = V2.search(p, size, cost, R=R, D=D, T=T, seed=seed, guard=guard, cover=cover)
    b = c_restore.search(p, size, cost, R=R, D=D, T=T, seed=seed, guard=guard, cover=cover)
    assert np.array_equal(a["root_n"], b["root_n"]) and np.array_equal(a["root_w"].view(np.uint32), b["root_w"].view(np.uint32))
    assert a["num_nodes"] == b["num_nodes"]
    # without covers the v2 search is the v1 search
    v1 = M.search(p, size, cost, R=R, D=D, T=T, seed=seed, guard=guard)
    v2 = V2.search(p, size, cost, R=R, D=D, T=T, seed=seed, guard=guard)
    assert np.array_equal(v1["root_n"], v2["root_n"]) and np.array_equal(v1["root_w"].view(np.uint32), v2["root_w"].view(np.uint32))


def test_exhaustive_small_optimum_prefers_restore():
    """Small instance: the exhaustive optimum holds the restore and none of the reversions it covers."""
    p, size, cost, cover = threshold_instance()
    A = 12
    p, size, cost, cover = p[:A], size[:A], cost[:A], cover[:A]
    cost = cost.copy(); cost[0] = 5.0                                   # cheap enough to win over 11 reversions
    st = _exhaustive(A, p, size, cost, None, cover)
    sc = V2.score(st, p, size, cost, None, cover)
    best = int(np.argmax(sc))
    assert best == 1
    assert list(itertools.compress(range(A), [(best >> a) & 1 for a in range(A)])) == [0]
