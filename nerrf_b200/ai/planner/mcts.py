"""ai.planner.mcts -- MCTS rollback planner (CUDA persistent leaf-parallel kernel, sm_90a).

Reference surface: ai/planner/mcts.py `search` (README.md:74,115; ROADMAP.md:84 -- named, never
written).  Behaviour: "500-1000 simulations", "Timeout: 5 min", input "Graph + anomaly scores +
predictions", output "Undo plan (file reversions, process kills)"
(docs/content/docs/architecture.mdx:62-72); candidates threat-model.mdx:205-223.
Frozen spec: DESIGN.md "MCTS spec" (leaf-parallel UCT, R rollouts per iteration, Philox RNG,
bit-exact integer statistics).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass

import numpy as np
import torch

from ... import _lib as L
from . import rewards as RW
from .rewards import Actions


@dataclass
class SearchResult:
    root_n: np.ndarray      # int32 [A]  rollouts through each root child
    root_w: np.ndarray      # fp32  [A]  sum of rollout values
    best: int               # recommended action (-1 if none)
    num_nodes: int
    lo: float
    inv_range: float
    rollouts: int

    @property
    def root_q(self):
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(self.root_n > 0, self.root_w / self.root_n.astype(np.float32), np.float32(0)).astype(np.float32)


def ln_table(T, R) -> np.ndarray:
    k = np.arange(T + 2, dtype=np.float64)
    k[0] = 1.0
    out = np.log(k * float(R)).astype(np.float32)
    out[0] = np.float32(0.0)
    return out


def best_child(root_n, root_w) -> int:
    """argmax over children with n > 0 of (n, Q, -a): robust child, Q breaks ties, then lowest index."""
    n = np.asarray(root_n); w = np.asarray(root_w, np.float32)
    if n.size == 0 or n.max() <= 0:
        return -1
    top = np.nonzero(n == n.max())[0]                         # most visited
    q = (w[top] / n[top].astype(np.float32)).astype(np.float32)
    return int(top[np.nonzero(q == q.max())[0][0]])           # highest Q among them, lowest index on ties


def merge_root_stats(results):
    """Root parallelism (SURVEY.md 8e): sum the per-tree root statistics in rank order."""
    n = np.zeros_like(results[0].root_n)
    w = np.zeros_like(results[0].root_w)
    for r in results:
        n = n + r.root_n
        w = (w + r.root_w).astype(np.float32)
    return n, w, best_child(n, w)


class SearchContext:
    """Device-resident state for repeated searches over the same candidate set (plan() re-roots up to
    `depth` times): the action arrays, ln table, tree workspace and pinned result buffers are allocated
    once; a search is then memset + one persistent kernel + one small D2H."""

    def __init__(self, actions: Actions, n_rollouts=4096, depth=50, iterations=64, c=math.sqrt(2.0), device=None):
        self.actions, self.R, self.D, self.T, self.c = actions, int(n_rollouts), int(depth), int(iterations), float(c)
        if self.R < 1 or (self.R & (self.R - 1)):
            raise ValueError("n_rollouts must be a power of two")
        self.device = torch.device(device or "cuda")
        if self.device.type != "cuda":
            raise L.NerrfError("mcts.search needs a CUDA device (no CPU fallback)")
        A = actions.A
        _, _, self.A_pad, self.nw = RW.layout(A)
        with torch.cuda.device(self.device):
            self.p, self.size, self.cost = actions.device_arrays(self.device)
            self.guard = actions.device_guard(self.device)
            self.cover = actions.device_cover(self.device)
            self.d_ln = torch.from_numpy(ln_table(self.T, self.R)).to(self.device)
            self.d_root = torch.empty(self.nw, device=self.device, dtype=torch.int32)
            # root_n | root_w | num_nodes in one buffer -> one D2H
            self.d_out = torch.empty(2 * self.A_pad + 1, device=self.device, dtype=torch.int32)
            self.h_out = torch.empty(2 * self.A_pad + 1, dtype=torch.int32).pin_memory()
            self.h_root = torch.empty(self.nw, dtype=torch.int32).pin_memory()
            need = C.c_size_t()
            L.check(L.lib().nerrf_mcts_workspace_bytes(A, self.T, self.R, C.byref(need)), "nerrf_mcts_workspace_bytes")
            self.ws_bytes = need.value
            self.ws = torch.empty(need.value, device=self.device, dtype=torch.uint8)

    def launch(self, seed=0, root_state=None, depth=None):
        """Enqueue one search on the current stream (asynchronous); returns (lo, inv_range)."""
        A = self.actions.A
        root = RW.empty_state(A) if root_state is None else (np.asarray(root_state, np.uint32) | RW.empty_state(A))
        lo, inv = RW.reward_bounds(self.actions, root)
        self.h_root.copy_(torch.from_numpy(root.view(np.int32)))
        self.d_root.copy_(self.h_root, non_blocking=True)
        o = self.d_out
        L.check(L.lib().nerrf_mcts_search_ex(L.ptr(self.p), L.ptr(self.size), L.ptr(self.cost), L.ptr(self.guard), L.ptr(self.cover),
                                             A, L.ptr(self.d_root), self.R,
                                          self.D if depth is None else int(depth), self.T, C.c_uint64(seed), self.c,
                                          float(lo), float(inv), L.ptr(self.d_ln), C.c_void_p(o.data_ptr()),
                                          C.c_void_p(o.data_ptr() + 4 * self.A_pad), C.c_void_p(o.data_ptr() + 8 * self.A_pad),
                                          L.ptr(self.ws), self.ws_bytes, L.current_stream_ptr()), "nerrf_mcts_search_ex")
        return float(lo), float(inv)

    def fetch(self, lo, inv) -> "SearchResult":
        self.h_out.copy_(self.d_out, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        A, Ap = self.actions.A, self.A_pad
        h = self.h_out.numpy()
        root_n = h[:A].copy(); root_w = h[Ap:Ap + A].view(np.float32).copy(); nn = int(h[2 * Ap])
        return SearchResult(root_n, root_w, best_child(root_n, root_w), nn, lo, inv, self.R * self.T)

    def search(self, seed=0, root_state=None, depth=None) -> "SearchResult":
        with torch.cuda.device(self.device):
            lo, inv = self.launch(seed, root_state, depth)
            return self.fetch(lo, inv)


class HostSession:
    """Host-buffer search handle (include/nerrf_b200.h nerrf_mcts_session_*): device buffers and a stream are allocated
    once; pass it as `host_call=` to search()."""

    def __init__(self, max_actions=1024, max_iterations=64, max_rollouts=4096, device=None):
        self.handle = C.c_void_p()
        dev = torch.device(device or "cuda")
        with torch.cuda.device(dev):
            L.check(L.lib().nerrf_mcts_session_create(int(max_actions), int(max_iterations), int(max_rollouts), C.byref(self.handle)),
                    "nerrf_mcts_session_create")

    def close(self):
        if self.handle:
            L.lib().nerrf_mcts_session_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def search(actions: Actions, scorer=None, n_rollouts: int = 4096, depth: int = 50, seed: int = 0,
           c: float = math.sqrt(2.0), iterations: int = 64, root_state=None, device=None, host_call: bool = False,
           context: SearchContext | None = None) -> SearchResult:
    """One tree search.  `scorer` must be None or ai.planner.rewards.score: the reward is evaluated
    inside the kernel (batched, R states per iteration).  host_call=True goes through the
    host-buffer C-ABI entry (copies inside the call; a HostSession instead of True reuses its device buffers).
    Pass a SearchContext to reuse device buffers on the device-pointer path."""
    if scorer is not None and scorer is not RW.score:
        raise NotImplementedError("the CUDA planner evaluates ai.planner.rewards.score in-kernel; "
                                  "custom scorers are not supported")
    A = actions.A
    NW, _, A_pad, nw = RW.layout(A)
    R, D, T = int(n_rollouts), int(depth), int(iterations)
    if R < 1 or (R & (R - 1)):
        raise ValueError("n_rollouts must be a power of two")
    if host_call:
        root = RW.empty_state(A) if root_state is None else (np.asarray(root_state, np.uint32) | RW.empty_state(A))
        lo, inv = RW.reward_bounds(actions, root)
        lnN = ln_table(T, R)
        root_n = np.zeros(A_pad, np.int32); root_w = np.zeros(A_pad, np.float32); nn = np.zeros(1, np.int32)
        as_p = lambda a: a.ctypes.data_as(C.c_void_p)
        gp = as_p(actions.guard) if actions.guard is not None else None
        cp = as_p(actions.cover) if actions.cover is not None else None
        if isinstance(host_call, HostSession):
            L.check(L.lib().nerrf_mcts_session_search_host_ex(host_call.handle, as_p(actions.p), as_p(actions.size), as_p(actions.cost),
                                                              gp, cp, A, as_p(root), R, D, T, C.c_uint64(seed), float(c), float(lo),
                                                              float(inv), as_p(lnN), as_p(root_n), as_p(root_w), as_p(nn)),
                    "nerrf_mcts_session_search_host_ex")
        else:
            L.check(L.lib().nerrf_mcts_search_host_ex(as_p(actions.p), as_p(actions.size), as_p(actions.cost), gp, cp, A, as_p(root), R,
                                                      D, T, C.c_uint64(seed), float(c), float(lo), float(inv), as_p(lnN), as_p(root_n),
                                                      as_p(root_w), as_p(nn)), "nerrf_mcts_search_host_ex")
        return SearchResult(root_n[:A].copy(), root_w[:A].copy(), best_child(root_n[:A], root_w[:A]), int(nn[0]),
                            float(lo), float(inv), R * T)
    ctx = context or SearchContext(actions, R, D, T, c, device)
    return ctx.search(seed, root_state, depth=D)


@dataclass
class Plan:
    actions: list           # committed action indices, in order
    scores: list            # exact rewards.score after each commit (scores[0] = initial state)
    searches: list          # SearchResult per step
    truncated: bool = False            # stopped at max_steps while an improving candidate still existed
    remaining_candidates: int = 0      # improving single actions left when the plan stopped (0 = complete)


def ranked_children(root_n, root_w):
    """Root children with n > 0 ordered by (n desc, Q desc, index asc) -- best_child() is element 0."""
    n = np.asarray(root_n); w = np.asarray(root_w, np.float32)
    idx = np.nonzero(n > 0)[0]
    q = (w[idx] / n[idx].astype(np.float32)).astype(np.float32)
    order = np.lexsort((idx, -q.astype(np.float64), -n[idx].astype(np.int64)))
    return idx[order]


class _DeviceCommit:
    """Buffers + call wrapper of nerrf_plan_commit (the validate-and-commit loop of plan() in one cooperative launch)."""

    def __init__(self, ctx: "SearchContext"):
        self.ctx = ctx
        dev = ctx.device
        need = C.c_size_t()
        L.check(L.lib().nerrf_plan_commit_workspace_bytes(4096, C.byref(need)), "nerrf_plan_commit_workspace_bytes")
        self.ws = torch.empty(need.value, device=dev, dtype=torch.uint8)
        self.ws_bytes = need.value
        self.d_state = torch.empty(ctx.nw, device=dev, dtype=torch.int32)
        self.d_cand = torch.empty(4096, device=dev, dtype=torch.int32)
        # actions | scores | n_out | state in one buffer -> one D2H per search
        self.cap = 4096
        self.d_out = torch.empty(2 * self.cap + 2 + ctx.nw, device=dev, dtype=torch.int32)
        self.h_out = torch.empty(2 * self.cap + 2 + ctx.nw, dtype=torch.int32).pin_memory()

    def run(self, state: np.ndarray, cand: np.ndarray, cur: float, max_commits: int, allow_tentative: bool):
        """-> (actions int list, scores float32 array, new state uint32 array, candidates left)."""
        ctx = self.ctx
        n = int(cand.shape[0])
        max_commits = min(int(max_commits), self.cap)
        with torch.cuda.device(ctx.device):
            self.d_cand[:n].copy_(torch.from_numpy(np.ascontiguousarray(cand, np.int32)), non_blocking=False)
            o = self.d_out
            st = o[2 * self.cap + 2:]
            st.copy_(torch.from_numpy(np.ascontiguousarray(state, np.uint32).view(np.int32)))
            L.check(L.lib().nerrf_plan_commit_ex(L.ptr(ctx.p), L.ptr(ctx.size), L.ptr(ctx.cost), L.ptr(ctx.guard), L.ptr(ctx.cover),
                                                 ctx.actions.A,
                                              C.c_void_p(st.data_ptr()), L.ptr(self.d_cand), n, C.c_float(cur), max_commits,
                                              int(bool(allow_tentative)), C.c_void_p(o.data_ptr()),
                                              C.c_void_p(o.data_ptr() + 4 * self.cap), C.c_void_p(o.data_ptr() + 8 * self.cap),
                                              L.ptr(self.ws), self.ws_bytes, L.current_stream_ptr()), "nerrf_plan_commit_ex")
            self.h_out.copy_(o, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        h = self.h_out.numpy()
        k = int(h[2 * self.cap])
        return (h[:k].tolist(), h[self.cap:self.cap + k].view(np.float32).copy(), h[2 * self.cap + 2:].view(np.uint32).copy(),
                int(h[2 * self.cap + 1]))


def _states_with(actions: Actions, rows) -> np.ndarray:
    st = np.repeat(RW.empty_state(actions.A)[None, :], len(rows), axis=0)
    for i, acts in enumerate(rows):
        for a_ in acts:
            st[i, a_ >> 5] |= np.uint32(1) << np.uint32(a_ & 31)
    return st


def _refine_restores(actions: Actions, out: "Plan", device):
    """Spec v2 clean-up of a finished plan (exact reward throughout; the plan order is kept, additions go last).
    (1) The commit loop is greedy: a restore that beats "nothing reverted" is committed even when reverting its files one by
    one would be better, and after it no reversion of those files can improve.  So each applied restore is compared with
    its alternative -- the plan without it plus every reversion it covers that improves that plan on its own -- and the
    better one is kept.  (2) A restore makes the reversions it covers pure downtime, but a reversion may have been
    committed before its restore: committed actions whose removal improves the reward are dropped (all at once when that
    is better still, else the best single one) until none is.  -> (final state, final score)."""
    score = lambda rows: RW.score(_states_with(actions, rows), actions, device=device).cpu().numpy()
    acts, cur = list(out.actions), np.float32(out.scores[-1])
    for r in [a_ for a_ in acts if (actions.cover == a_).any()]:
        base = [a_ for a_ in acts if a_ != r]
        cov = [int(a_) for a_ in np.nonzero(actions.cover == r)[0] if int(a_) not in base]
        if not cov:
            continue
        sc = score([base] + [base + [a_] for a_ in cov])
        alt = base + [a_ for a_, v in zip(cov, sc[1:]) if v > sc[0]]
        s_alt = score([alt])[0]
        if s_alt > cur:
            acts, cur = alt, s_alt
    while len(acts) > 1:
        sc = score([acts[:i] + acts[i + 1:] for i in range(len(acts))])
        better = sc > cur
        if not better.any():
            break
        rest = [a_ for a_, b in zip(acts, better) if not b]
        s_all = score([rest])[0]
        k = int(np.argmax(sc))
        if s_all >= sc[k]:
            acts, cur = rest, s_all
        else:
            acts, cur = acts[:k] + acts[k + 1:], sc[k]
    if acts != list(out.actions):
        pref = score([acts[:i] for i in range(1, len(acts) + 1)])
        out.actions, out.scores = acts, out.scores[:1] + [float(v) for v in pref]
    return _states_with(actions, [out.actions])[0], float(out.scores[-1])


def plan(actions: Actions, max_steps: int | None = None, n_rollouts: int = 4096, depth: int = 50, seed: int = 0,
         c: float = math.sqrt(2.0), iterations: int = 64, device=None, commit_per_search: int = 1, merge=None,
         lookahead: bool | None = None, patience: int = 8, device_commit: bool = True) -> Plan:
    """Undo plan = repeated search / commit / re-root.  Each step the search ranks the root
    children; the candidates are then VALIDATED with the exact reward (one batched
    rewards.score call over all candidate next-states, mirroring the reference's "sandbox
    validates, then apply" gate, architecture.mdx:81-86): the highest-ranked candidate whose
    exact reward improves on the current state is committed; the plan ends when none does.

    commit_per_search > 1: after a search, up to that many ranked candidates are committed, each one re-validated
    with the exact reward against the state INCLUDING the commits before it (large incidents: thousands of files
    would otherwise need one tree search per file).
    merge: root parallelism over several GPUs -- a callable (root_n, root_w) -> (root_n, root_w) that sums the root
    statistics of all ranks in rank order (nerrf_b200.dist); every rank then takes identical decisions.
    lookahead (default: on when the actions carry guards (spec v1) or covers (spec v2)): the reward is then not separable --
    killing a process costs downtime and only pays off through the reversions it makes durable, a restore costs downtime
    and makes the reversions it covers redundant -- so a step that no single action improves
    is not the end: the search's recommended child is committed TENTATIVELY, planning continues from there for at most
    `patience` steps below the best reward seen, and the plan is finally cut back to its best prefix (what the sandbox
    would approve).
    With covers (spec v2) the finished plan is refined with the exact reward (_refine_restores): each applied restore is
    weighed against reverting its files one by one, and committed actions whose removal improves the reward (a reversion
    committed before the restore that covers it) are dropped.
    device_commit (default): the validate-and-commit loop runs on the device in one launch per search (nerrf_plan_commit);
    False keeps it as a host loop over rewards.score calls -- the same decisions bit for bit (tests compare the two)."""
    A = actions.A
    state = RW.empty_state(A)
    max_steps = A if max_steps is None else max_steps          # a plan may need every candidate; `depth` is the ROLLOUT horizon
    cur = float(RW.score(state[None, :], actions, device=device).cpu()[0])
    out = Plan([], [cur], [])
    ctx = SearchContext(actions, n_rollouts, depth, iterations, c, device)
    dc = None
    step = 0
    lookahead = (actions.guard is not None or actions.cover is not None) if lookahead is None else lookahead
    best_score, best_len = cur, 0
    while len(out.actions) < max_steps:
        # one-commit-per-search plans keep a total horizon of `depth` moves; batch-committing plans (large incidents)
        # search with the full rollout horizon every time
        res = ctx.search(seed + step, state, depth=max(depth - len(out.actions), 1) if commit_per_search == 1 else depth)
        step += 1
        if merge is not None:
            n, w = merge(res.root_n, res.root_w)
            res = SearchResult(n, w, best_child(n, w), res.num_nodes, res.lo, res.inv_range, res.rollouts)
        out.searches.append(res)
        cand = ranked_children(res.root_n, res.root_w)
        if cand.size == 0:
            break
        committed = 0
        if device_commit:
            # the validate-and-commit loop below as ONE cooperative launch (nerrf_plan_commit): same decisions, same scores
            dc = dc if dc is not None else _DeviceCommit(ctx)
            acts, scs, state, _left = dc.run(state, cand, cur, min(commit_per_search, max_steps - len(out.actions)),
                                             lookahead and len(out.actions) - best_len < patience)
            for a_, s_ in zip(acts, scs.tolist()):
                cur = float(s_)
                out.actions.append(int(a_)); out.scores.append(cur)
                committed += 1
                if cur > best_score:
                    best_score, best_len = cur, len(out.actions)
            cand = cand[:0]
        while cand.size and committed < commit_per_search and len(out.actions) < max_steps:
            nxt = np.repeat(state[None, :], cand.size, axis=0)
            nxt[np.arange(cand.size), cand >> 5] |= (np.uint32(1) << (cand & 31).astype(np.uint32)).astype(np.uint32)
            sc = RW.score(nxt, actions, device=device).cpu().numpy()
            better = np.nonzero(sc > np.float32(cur))[0]
            if better.size == 0:
                if lookahead and committed == 0 and len(out.actions) - best_len < patience:
                    better = np.zeros(1, np.int64)                       # tentative: the search's recommendation
                else:
                    break
            k = int(better[0])
            state, cur = nxt[k].copy(), float(sc[k])
            out.actions.append(int(cand[k])); out.scores.append(cur)
            committed += 1
            if cur > best_score:
                best_score, best_len = cur, len(out.actions)
            cand = cand[better[1:]] if commit_per_search > 1 else cand[:0]     # only candidates that still looked improving
        if committed == 0 or (lookahead and len(out.actions) - best_len >= patience):
            break
    if len(out.actions) > best_len:                                      # drop a tentative tail that never paid off
        out.actions = out.actions[:best_len]; out.scores = out.scores[:best_len + 1]
        state = RW.empty_state(A)
        for a_ in out.actions:
            state[a_ >> 5] |= np.uint32(1) << np.uint32(a_ & 31)
        cur = best_score
    if actions.cover is not None and out.actions:
        state, cur = _refine_restores(actions, out, device)
    if len(out.actions) >= max_steps and len(out.actions) < A:
        # step limit hit: say so instead of handing back a silently incomplete plan (one batched exact-reward call)
        rest = np.array([a for a in range(A) if not (state[a >> 5] >> np.uint32(a & 31)) & np.uint32(1)], np.int64)
        if rest.size:
            nxt = np.repeat(state[None, :], rest.size, axis=0)
            nxt[np.arange(rest.size), rest >> 5] |= (np.uint32(1) << (rest & 31).astype(np.uint32)).astype(np.uint32)
            sc = RW.score(nxt, actions, device=device).cpu().numpy()
            out.remaining_candidates = int((sc > np.float32(cur)).sum())
            out.truncated = out.remaining_candidates > 0
    return out
