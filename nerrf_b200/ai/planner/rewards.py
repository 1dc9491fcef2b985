"""ai.planner.rewards -- rollback reward scorer (CUDA, sm_90a).

Reference surface: ai/planner/rewards.py (README.md:74 -- named, never written).
Behaviour: `Reward = -(data_loss + 0.1 x downtime)` (README.md:115); "restoration gain - side
effects" (docs/content/docs/architecture.mdx:71); candidate cost/confidence example
(threat-model.mdx:205-223).  Frozen spec: SURVEY.md 8a row a6 / DESIGN.md "Reward spec":

    data_loss(s) = sum_{a not in s} p_a size_a + sum_{a in s} (1-p_a) size_a ;  downtime(s) = sum_{a in s} cost_a
    score(s) = -(data_loss + 0.1 downtime)            fp32, fixed association order (bit-exact)

Spec v1 (DESIGN.md 1.3) adds the one non-separable term the reference's own candidate list implies
(threat-model.mdx:208-222: "Reverse file encryption" next to "Kill process python3"): every action may name a GUARD
-- the index (< 32) of the "kill process" action of the process that wrote its file.  An applied action whose guard
is NOT applied additionally loses w_a = p_guard * p_a * size_a: the live process re-encrypts the reverted file.

Spec v2 (DESIGN.md 1.3) gives the third candidate kind, "Restore from backup" (threat-model.mdx:216-219), its meaning:
every action may name a COVER -- the index (< 32) of the restore action of the directory that holds its file.  An
action that is not applied but whose cover is applied is restored all the same: it loses (1-p_a) size_a (plus w_a while
its guard lives), like an applied action, but adds no downtime.  A restore action itself has p = 0 and size = the
collateral it destroys (u = 0, v = collateral).

States are bitsets: uint32 [B, n_words], action a = bit (a & 31) of word (a >> 5),
n_words = 32*NW with NW = 1/2/4 for A <= 1024/2048/4096.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch

from ... import _lib as L

KIND_REVERT, KIND_KILL, KIND_RESTORE = 0, 1, 2
KIND_COST = {KIND_REVERT: 1.0, KIND_KILL: 10.0, KIND_RESTORE: 100.0}     # threat-model.mdx:210,214,218


@dataclass
class Actions:
    """Undo candidates.  p = probability the target is attack damage (from GraphSAGE_T / lstm),
    size = MB at stake, cost = seconds of downtime if applied."""
    p: np.ndarray
    size: np.ndarray
    cost: np.ndarray
    kind: np.ndarray | None = None
    names: list = field(default_factory=list)
    guard: np.ndarray | None = None      # int32 [A]: index (< 32) of the kill action guarding a, or -1 (spec v1)
    cover: np.ndarray | None = None      # int32 [A]: index (< 32) of the restore action covering a, or -1 (spec v2)

    def __post_init__(self):
        self.p = np.ascontiguousarray(_np(self.p), dtype=np.float32)
        self.size = np.ascontiguousarray(_np(self.size), dtype=np.float32)
        self.cost = np.ascontiguousarray(_np(self.cost), dtype=np.float32)
        if not (self.p.shape == self.size.shape == self.cost.shape and self.p.ndim == 1):
            raise ValueError("p, size, cost must be 1-D arrays of equal length")
        if not 1 <= self.p.shape[0] <= 4096:
            raise ValueError("number of actions must be in 1..4096")
        if self.guard is not None:
            g = np.ascontiguousarray(_np(self.guard), dtype=np.int32)
            if g.shape != self.p.shape or (g < -1).any() or (g >= 32).any() or (g >= self.p.shape[0]).any():
                raise ValueError("guard must be -1 or the index (< 32, < A) of the kill action, one per action")
            self.guard = g if (g >= 0).any() else None
        if self.cover is not None:
            self.cover = check_cover(self.cover, self.guard, self.p.shape[0])

    @property
    def A(self):
        return self.p.shape[0]

    @classmethod
    def from_scores(cls, anomaly_score, encrypt_probability, size, kind, names=None):
        """p_a = (anomaly_score_a + encrypt_probability_a) / 2  (SURVEY.md 8a a6)."""
        p = 0.5 * (_np(anomaly_score).astype(np.float32) + _np(encrypt_probability).astype(np.float32))
        kind = _np(kind).astype(np.int64)
        cost = np.vectorize(KIND_COST.get)(kind).astype(np.float32)
        return cls(p, size, cost, kind, list(names or []))

    def device_arrays(self, device):
        return tuple(torch.from_numpy(a).to(device) for a in (self.p, self.size, self.cost))

    def device_guard(self, device):
        return None if self.guard is None else torch.from_numpy(self.guard).to(device)

    def device_cover(self, device):
        return None if self.cover is None else torch.from_numpy(self.cover).to(device)


def check_cover(cover, guard, A):
    """Validated int32 [A] cover table, or None when no action is covered.  cover[a] is -1 or the index of a restore action
    in state word 0 (< 32, < A), never a itself; a restore action is not covered itself (one level) and is no guard target."""
    c = np.ascontiguousarray(_np(cover), dtype=np.int32)
    if c.shape != (A,):
        raise ValueError("cover must hold one entry per action")
    if (c < -1).any() or (c >= min(32, A)).any():
        raise ValueError("cover must be -1 or the index (< 32, < A) of the restore action, one per action")
    if (c == np.arange(A)).any():
        raise ValueError("an action cannot cover itself")
    targets = np.unique(c[c >= 0])
    if (c[targets] >= 0).any():
        raise ValueError("a restore action cannot itself be covered (covers do not chain)")
    if guard is not None and np.isin(targets, guard[guard >= 0]).any():
        raise ValueError("an action cannot be both a guard and a cover target")
    return c if targets.size else None


def _np(a):
    return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def layout(A):
    """-> (NW, chunk, A_pad, n_words)"""
    if A < 1 or A > 4096:
        raise ValueError("number of actions must be in 1..4096")
    NW = 1 if A <= 1024 else (2 if A <= 2048 else 4)
    return NW, 32 * NW, 1024 * NW, 32 * NW


def empty_state(A) -> np.ndarray:
    """Bitset with no action applied (padding bits a >= A are set: never legal)."""
    _, _, A_pad, nw = layout(A)
    s = np.zeros(nw, np.uint32)
    for a in range(A, min(A_pad, ((A + 31) // 32) * 32)):
        s[a >> 5] |= np.uint32(1) << np.uint32(a & 31)
    s[(A + 31) // 32:] = np.uint32(0xFFFFFFFF)
    return s


def pack_states(applied, A=None) -> np.ndarray:
    """bool [B, A] (or list of index lists) -> uint32 [B, n_words]."""
    if isinstance(applied, (list, tuple)) and (len(applied) == 0 or not isinstance(applied[0], (bool, np.bool_))):
        assert A is not None
        m = np.zeros((len(applied), A), bool)
        for i, idx in enumerate(applied):
            m[i, list(idx)] = True
        applied = m
    applied = np.asarray(applied, bool)
    B, A_ = applied.shape
    _, _, A_pad, nw = layout(A_)
    bits = np.ones((B, A_pad), bool)
    bits[:, :A_] = applied
    sh = np.arange(32, dtype=np.uint64)
    return (bits.reshape(B, nw, 32).astype(np.uint64) << sh).sum(axis=2).astype(np.uint32)


def score(states, actions: Actions, device=None) -> torch.Tensor:
    """states uint32 [B, n_words] (numpy, or a CUDA int32/uint32-viewed tensor) -> fp32 [B] on the device."""
    if isinstance(states, torch.Tensor):
        st = states
        device = st.device
    else:
        device = torch.device(device or "cuda")
        st = torch.from_numpy(np.ascontiguousarray(states, dtype=np.uint32).view(np.int32)).to(device)
    if device.type != "cuda":
        raise L.NerrfError("rewards.score needs a CUDA device (no CPU fallback)")
    _, _, _, nw = layout(actions.A)
    st = st.contiguous().view(-1, nw)
    B = st.shape[0]
    p, size, cost = actions.device_arrays(device)
    guard = actions.device_guard(device)
    cover = actions.device_cover(device)
    out = torch.empty(B, device=device, dtype=torch.float32)
    with torch.cuda.device(device):
        L.check(L.lib().nerrf_reward_score_ex(L.ptr(st), B, L.ptr(p), L.ptr(size), L.ptr(cost), L.ptr(guard), L.ptr(cover),
                                              actions.A, L.ptr(out), L.current_stream_ptr()), "nerrf_reward_score_ex")
    return out


def reward_bounds(actions: Actions, root_state=None):
    """(lo, inv_range): worst score over supersets of root_state and 1/(best - worst), so that
    value = (score - lo) * inv_range is in ~[0,1] for UCT.  float64 with exactly-rounded
    summation (math.fsum), then rounded to fp32.  With covers (spec v2) an action that is not applied may still be
    restored by its cover: its best case is then min(u, v, v + 0.1 cost), its worst case still includes vw."""
    A = actions.A
    p = actions.p; one = np.float32(1.0)
    u = (p * actions.size).astype(np.float32).astype(np.float64)
    v = ((one - p).astype(np.float32) * actions.size).astype(np.float32).astype(np.float64)
    applied_cost = v + 0.1 * actions.cost.astype(np.float64)
    applied_worst = applied_cost
    if actions.guard is not None:            # an applied action may also pay its guard penalty: a valid (not tight) bound
        g = actions.guard.astype(np.int64)
        u32 = (p * actions.size).astype(np.float32); v32 = ((one - p).astype(np.float32) * actions.size).astype(np.float32)
        w32 = (np.where(g >= 0, p[np.maximum(g, 0)], np.float32(0.0)).astype(np.float32) * u32).astype(np.float32)
        vw = np.where(g >= 0, (v32 + w32).astype(np.float32), v32).astype(np.float64)
        applied_worst = vw + 0.1 * actions.cost.astype(np.float64)
    fixed = np.zeros(A, bool)
    if root_state is not None:
        rs = np.asarray(root_state, np.uint32)
        idx = np.arange(A)
        fixed = ((rs[idx >> 5] >> (idx & 31).astype(np.uint32)) & np.uint32(1)) != 0
    worst = np.where(fixed, applied_worst, np.maximum(u, applied_worst))
    best = np.where(fixed, applied_cost, np.minimum(u, applied_cost))
    if actions.cover is not None:              # a covered action may be restored without being applied: loss v, no downtime
        best = np.where(~fixed & (actions.cover >= 0), np.minimum(best, v), best)
    lo = np.float32(-math.fsum(worst.tolist()))
    hi = -math.fsum(best.tolist())
    rng = hi - float(lo)
    inv = np.float32(1.0) if not (rng > 0.0) else np.float32(1.0 / rng)
    return lo, inv
