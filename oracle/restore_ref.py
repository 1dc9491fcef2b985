"""Planner spec v2 oracle (numpy, bit-exact fp32; test infra -- see oracle/__init__.py): rewards with COVER actions.

Spec v1 (rewards_ref.py) gave "Kill process" a meaning; spec v2 gives the third candidate kind of the reference's list,
"Restore from backup" (cost 100, confidence 1.0; docs/content/docs/threat-model.mdx:205-223).  A restore action brings
back every file of one directory from the pre-attack snapshot, so one restore can stand in for many file reversions
(the 1000+-file encryption loop of architecture.mdx:104-108).

Every action a may name a COVER c = cover_a in 0..31 -- the index of the restore action of its directory (restores live
in state word 0, next to the kills) -- or -1.  For a state s:
    restored_a = a in s  or  (cover_a >= 0 and cover_a in s)
    alive_a    = guard_a >= 0 and guard_a not in s
    data-loss term of a = restored_a ? (alive_a ? vw_a : v_a) : u_a
    downtime term of a  = a in s ? cost_a : 0
Summation order, layout and rounding are spec v1's exactly (one term per action per sum, lane-sequential, xor
butterfly); cover = None is spec v1 bit for bit.  Validity: cover_a in {-1} U [0, min(32, A)), cover_a != a, a cover
target is not covered itself, and no index is both a guard and a cover target.

This module reuses spec v1's layout helpers and the v1 search's random choices (the rollout policy does not depend on the
reward), and restates only what the covers change.
"""
import math

import numpy as np

from . import mcts_ref as M
from . import rewards_ref as RW

F32 = np.float32


def check_cover(cover, guard, A):
    """-> int64 [A_pad] cover table (-1 = none); ValueError on an invalid table."""
    _, _, A_pad, _ = RW.layout(A)
    out = np.full(A_pad, -1, np.int64)
    if cover is None:
        return out
    c = np.asarray(cover, np.int64)
    if c.shape != (A,):
        raise ValueError("cover must hold one entry per action")
    if (c < -1).any() or (c >= min(32, A)).any():
        raise ValueError("cover must be -1 or the index (< 32, < A) of the restore action")
    if (c == np.arange(A)).any():
        raise ValueError("an action cannot cover itself")
    targets = np.unique(c[c >= 0])
    if (c[targets] >= 0).any():
        raise ValueError("a restore action cannot itself be covered")
    if guard is not None:
        g = np.asarray(guard, np.int64)
        if np.isin(targets, g[g >= 0]).any():
            raise ValueError("an action cannot be both a guard and a cover target")
    out[:A] = c
    return out


def score(states, p, size, cost, guard=None, cover=None):
    """states uint32 [B, n_words] -> fp32 [B] (spec v2)."""
    A = np.asarray(p).shape[0]
    NW, chunk, A_pad, nw = RW.layout(A)
    states = np.asarray(states, dtype=np.uint32).reshape(-1, nw)
    u, v, c = RW.action_terms(p, size, cost)
    cv = check_cover(cover, guard, A)
    applied = RW.unpack_bits(states)
    g, vw = RW.guard_terms(p, size, cost, guard)
    alive = (g[None, :] >= 0) & ~applied[:, np.maximum(g, 0)]
    restored = applied | ((cv[None, :] >= 0) & applied[:, np.maximum(cv, 0)])
    v_eff = np.where(alive, vw[None, :], v[None, :]).astype(F32)
    dl_terms = np.where(restored, v_eff, u[None, :]).astype(F32)
    dt_terms = np.where(applied, c[None, :], F32(0.0)).astype(F32)
    dl = RW._lane_tree_sum(dl_terms, chunk)
    dt = RW._lane_tree_sum(dt_terms, chunk)
    tenth = (F32(0.1) * dt).astype(F32)
    return (-((dl + tenth).astype(F32))).astype(F32)


def reward_bounds(p, size, cost, root_state=None, guard=None, cover=None):
    """(lo, inv_range) as RW.reward_bounds, still a valid bound with covers: an action that is not applied but covered
    can cost v with no downtime, so its best case is min(u, v, v + 0.1 cost); the worst case still includes vw."""
    A = np.asarray(p).shape[0]
    cv = check_cover(cover, guard, A)[:A]
    u, v, c = RW.action_terms(p, size, cost)
    u = u.astype(np.float64)[:A]; v = v.astype(np.float64)[:A]; c = c.astype(np.float64)[:A]
    applied_cost = v + 0.1 * c
    _, vw = RW.guard_terms(p, size, cost, guard)
    applied_worst = vw.astype(np.float64)[:A] + 0.1 * c
    if root_state is None:
        fixed = np.zeros(A, bool)
    else:
        fixed = RW.unpack_bits(np.asarray(root_state, np.uint32)[None, :])[0][:A]
    worst = np.where(fixed, applied_worst, np.maximum(u, applied_worst))
    best = np.where(fixed, applied_cost, np.minimum(u, applied_cost))
    best = np.where(~fixed & (cv >= 0), np.minimum(best, v), best)
    lo = -math.fsum(worst.tolist())
    hi = -math.fsum(best.tolist())
    lo32 = F32(lo)
    rng = hi - float(lo32)
    inv = F32(1.0) if not (rng > 0.0) else F32(1.0 / rng)
    return lo32, inv


def rollouts(s0, depth, t, R, D, seed, p, size, cost, lo, inv_range, guard=None, cover=None):
    """One leaf evaluation (see mcts_ref.rollouts): the same random states, valued with the spec-v2 reward."""
    _, first, L0, s = M.rollouts(s0, depth, t, R, D, seed, p, size, cost, lo, inv_range, guard)
    sc = score(s, p, size, cost, guard, cover)
    val = ((sc - F32(lo)).astype(F32) * F32(inv_range)).astype(F32)
    return val, first, L0, s


def search(p, size, cost, R=4096, D=50, T=64, seed=0, c=np.sqrt(2.0), root_state=None, bounds=None, guard=None,
           cover=None):
    """mcts_ref.search with the spec-v2 reward: same tree policy, same backup order."""
    p = np.asarray(p, F32); size = np.asarray(size, F32); cost = np.asarray(cost, F32)
    A = p.shape[0]
    NW, chunk, A_pad, nw = RW.layout(A)
    assert R >= 1 and (R & (R - 1)) == 0, "R must be a power of two"
    root = RW.empty_state(A) if root_state is None else (np.asarray(root_state, np.uint32) | RW.empty_state(A))
    lo, inv = reward_bounds(p, size, cost, root, guard, cover) if bounds is None else bounds
    lnN = M.ln_table(T, R)
    c32 = F32(c)
    tree = M.Tree(T, A_pad)
    for t in range(T):
        node = 0; state = root.copy(); depth = 0; path = []
        while tree.visits[node] > 0:
            legal = ~RW.unpack_bits(state[None, :])[0]
            if depth >= D or not legal.any():
                break
            n = tree.child_n[node]
            nf = n.astype(F32)
            with np.errstate(divide="ignore", invalid="ignore"):
                q = (tree.child_w[node] / nf).astype(F32)
                ratio = (lnN[tree.visits[node]] / nf).astype(F32)
                key = (q + (c32 * np.sqrt(ratio).astype(F32)).astype(F32)).astype(F32)
            key = np.where(n == 0, F32(np.inf), key)
            key = np.where(legal, key, -np.inf)
            a = int(np.argmax(key))
            path.append((node, a))
            state[a >> 5] |= np.uint32(1) << np.uint32(a & 31)
            depth += 1
            if tree.child_id[node][a] == -1:
                nid = tree.num_nodes
                tree.num_nodes += 1
                tree.child_id[node][a] = nid
                node = nid
                break
            node = int(tree.child_id[node][a])
        leaf = node
        val, first, L0, _ = rollouts(state, depth, t, R, D, seed, p, size, cost, lo, inv, guard, cover)
        total = M.tree_sum(val)
        if first[0] >= 0:
            for q_ in range(min(R, L0)):
                a = int(first[q_])
                idx = np.arange(q_, R, L0)
                w = tree.child_w[leaf][a]
                for i in idx:
                    w = F32(w + val[i])
                tree.child_w[leaf][a] = w
                tree.child_n[leaf][a] += len(idx)
        tree.visits[leaf] += 1
        for (nd, a) in path:
            tree.child_n[nd][a] += R
            tree.child_w[nd][a] = F32(tree.child_w[nd][a] + total)
            tree.visits[nd] += 1
    root_n = tree.child_n[0][:A].copy()
    root_w = tree.child_w[0][:A].copy()
    return {"root_n": root_n, "root_w": root_w, "best": M.best_child(root_n, root_w), "num_nodes": tree.num_nodes,
            "lo": lo, "inv_range": inv}
