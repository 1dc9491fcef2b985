"""Planner spec v2 timing: the MCTS search and the plan-commit loop at the BASELINE cfg-3 shape (A = 1024, R = 4096, D = 50,
16 iterations), with and without cover (restore) actions.

    python scripts/restore_timing.py --out result.json [--baseline-lib path/to/older/libnerrf_b200.so]

Cases, timed with CUDA events on one stream:
  * no covers, this build (`nerrf_mcts_search`) -- and, with --baseline-lib, the same call into an older build of the
    library, alternated round by round with this one so both see the same clocks;
  * 8 restore slots (actions 0..7) covering 900 of the other actions (`nerrf_mcts_search_ex`).
For each case: rollouts/s of the search (R * T / search time) and the time of one plan-commit launch over the search's
ranked root children (up to 64 commits).  Root statistics are digested, so equal digests mean the same bits.  The card's
name, power limit and SM clock (NVML) are recorded with the numbers."""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nerrf_b200 import _lib as L                      # noqa: E402
from nerrf_b200.ai.planner import mcts, rewards      # noqa: E402
from nerrf_b200.ai.planner.rewards import Actions    # noqa: E402

A, R, D, T = 1024, 4096, 50, 16


def card_info():
    import pynvml as nv
    nv.nvmlInit()
    h = nv.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
    name = nv.nvmlDeviceGetName(h)
    return {"name": name.decode() if isinstance(name, bytes) else name,
            "power_limit_w": nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
            "sm_clock_mhz": nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM),
            "sm_clock_max_mhz": nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)}


def actions(with_cover):
    rng = np.random.default_rng(0)
    p = rng.beta(0.5, 0.5, A).astype(np.float32)
    size = rng.lognormal(np.log(2.0), 1.0, A).astype(np.float32)
    cost = rng.choice([1.0, 10.0, 100.0], A, p=[.9, .09, .01]).astype(np.float32)
    cover = None
    if with_cover:
        p[:8] = 0.0; size[:8] = rng.uniform(0.0, 20.0, 8).astype(np.float32); cost[:8] = 100.0
        cover = np.full(A, -1, np.int32)
        idx = 8 + rng.permutation(A - 8)[:900]
        cover[idx] = rng.integers(0, 8, 900)
    return Actions(p, size, cost, cover=cover)


def bind(h):
    V = C.c_void_p
    h.nerrf_mcts_search.argtypes = [V, V, V, V, C.c_int, V, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_float, C.c_float, C.c_float,
                                    V, V, V, V, V, C.c_size_t, V]
    h.nerrf_plan_commit.argtypes = [V, V, V, V, C.c_int, V, V, C.c_int, C.c_float, C.c_int, C.c_int, V, V, V, V, C.c_size_t, V]
    return h


class Case:
    """Device buffers of one search + commit on `act`, callable through the plain (no-cover) symbols of any build of the
    library or through this build's *_ex symbols."""

    def __init__(self, act):
        dev = torch.device("cuda")
        self.act = act
        self.p, self.size, self.cost = act.device_arrays(dev)
        self.cover = act.device_cover(dev)
        self.lo, self.inv = rewards.reward_bounds(act)
        self.ln = torch.from_numpy(mcts.ln_table(T, R)).to(dev)
        self.root = torch.from_numpy(rewards.empty_state(A).view(np.int32)).to(dev)
        self.rn = torch.zeros(1024, dtype=torch.int32, device=dev)
        self.rw = torch.zeros(1024, dtype=torch.float32, device=dev)
        self.nn = torch.zeros(1, dtype=torch.int32, device=dev)
        need = C.c_size_t()
        L.check(L.lib().nerrf_mcts_workspace_bytes(A, T, R, C.byref(need)))
        self.ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        L.check(L.lib().nerrf_plan_commit_workspace_bytes(4096, C.byref(need)))
        self.cws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        self.state = torch.empty(32, dtype=torch.int32, device=dev)
        self.cand = torch.empty(4096, dtype=torch.int32, device=dev)
        self.out = torch.empty(2 * 64 + 2, dtype=torch.int32, device=dev)
        self.cur = float(rewards.score(rewards.empty_state(A)[None, :], act).cpu()[0])

    def search(self, h, ex):
        P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        args = [P(self.root), R, D, T, C.c_uint64(7), np.sqrt(2.0), float(self.lo), float(self.inv), P(self.ln), P(self.rn),
                P(self.rw), P(self.nn), P(self.ws), self.ws.numel(), L.current_stream_ptr()]
        if ex:
            rc = h.nerrf_mcts_search_ex(P(self.p), P(self.size), P(self.cost), None, P(self.cover), A, *args)
        else:
            rc = h.nerrf_mcts_search(P(self.p), P(self.size), P(self.cost), None, A, *args)
        assert rc == 0, h.nerrf_last_error()

    def commit(self, h, ex, cand):
        P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        n = int(cand.shape[0])
        self.cand[:n].copy_(torch.from_numpy(cand.astype(np.int32)))
        self.state.copy_(self.root)
        o = self.out.data_ptr()
        args = [P(self.state), P(self.cand), n, C.c_float(self.cur), 64, 0, C.c_void_p(o), C.c_void_p(o + 4 * 64),
                C.c_void_p(o + 8 * 64), P(self.cws), self.cws.numel(), L.current_stream_ptr()]
        if ex:
            rc = h.nerrf_plan_commit_ex(P(self.p), P(self.size), P(self.cost), None, P(self.cover), A, *args)
        else:
            rc = h.nerrf_plan_commit(P(self.p), P(self.size), P(self.cost), None, A, *args)
        assert rc == 0, h.nerrf_last_error()

    def timed(self, fn, reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn()                                                               # warm-up (smem opt-in, caches)
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            e0.record(); fn(); e1.record(); e1.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.median(ts))

    def run(self, h, ex, reps):
        ms = self.timed(lambda: self.search(h, ex), reps)
        rn, rw = self.rn.cpu().numpy(), self.rw.cpu().numpy()
        digest = hashlib.sha256(rn.tobytes() + rw.tobytes()).hexdigest()[:16]
        cand = mcts.ranked_children(rn[:A], rw[:A])
        cms = self.timed(lambda: self.commit(h, ex, cand), reps)
        return {"search_ms": ms, "rollouts_per_s": R * T / (ms * 1e-3), "commit_ms": cms, "n_candidates": int(cand.size),
                "root_digest": digest}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--baseline-lib", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    new = bind(L.lib())
    old = bind(C.CDLL(a.baseline_lib)) if a.baseline_lib else None
    plain, covered = Case(actions(False)), Case(actions(True))
    res = {"shape": {"A": A, "R": R, "D": D, "T": T, "cover_slots": 8, "covered_actions": 900}, "card_before": card_info(),
           "rounds": []}
    for r in range(a.rounds):
        row = {}
        order = [("baseline", old), ("this", new)] if r % 2 == 0 else [("this", new), ("baseline", old)]
        for name, h in order:
            if h is not None:
                row[name + "_no_cover"] = plain.run(h, False, a.reps)
        row["this_cover"] = covered.run(new, True, a.reps)
        res["rounds"].append(row)
        print(json.dumps(row), flush=True)
    res["card_after"] = card_info()
    summary = {}
    for k in res["rounds"][0]:
        v = [row[k]["rollouts_per_s"] for row in res["rounds"]]
        c = [row[k]["commit_ms"] for row in res["rounds"]]
        summary[k] = {"rollouts_per_s_median": float(np.median(v)), "rollouts_per_s_min": min(v), "rollouts_per_s_max": max(v),
                      "commit_ms_median": float(np.median(c)), "digests": sorted({row[k]["root_digest"] for row in res["rounds"]})}
    res["summary"] = summary
    print(json.dumps(summary, indent=1))
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
