"""End-to-end detection -> planning pipeline on one GPU (BASELINE config 5 in miniature / at scale).

    events (EventBatch / TRACE json) --graph.py--> temporal graph --GraphSAGE_T--> node anomaly scores
      --> top-A candidate file nodes --lstm--> encrypt_probability --rewards.Actions--> mcts.plan --> undo plan

Reference anchors: the intended stack of docs/content/docs/architecture.mdx:12-86 (graph constructor ->
AI models -> planner -> sandbox) and threat-model.mdx:141-223 (phases 2-5).  Everything on the hot path runs
through the C-ABI kernels; the host side here is glue + timing.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field

import numpy as np
import torch

from . import graph as G
from .ai.models import GraphSAGE_T, lstm
from .ai.planner import mcts
from .ai.planner.rewards import Actions, KIND_KILL as RW_KIND_KILL, KIND_RESTORE as RW_KIND_RESTORE, KIND_COST

_SEQ_EVENT_SLOT = {"file_created": 0, "file_encrypt_start": 1, "file_encrypt_complete": 2, "ransom_note_created": 3,
                   "openat": 4, "write": 5, "rename": 6}


def file_sequences(events, g: G.TemporalGraph, t_max=lstm.T_MAX, observable=False, return_events=False):
    """Per-file event sequences for the LSTM (the last `t_max` events of each file node, oldest first).
    Features (D_in = 16, named by lstm.FEATURE_NAMES): one-hot event kind (8), log1p(size)/20, dt to the previous event of
    the file (s, clipped), time since trace start / window, .lockbit flag, /tmp|/proc flag, 3 spare (the simulator's
    `phase` annotation is ground truth, not an observable: it is deliberately NOT a feature, so wire-format traces give
    the same sequences).  return_events: a fourth array, int64 [n_files, t_max], the event of each step as an index into
    graph.resolve_event_paths(events) (the ids graph_from_events' meta["edge_event"] / meta["event_info"] use), -1 at
    padded steps."""
    merge = g.meta.get("merge_renames", True)
    keys = g.meta.get("file_keys")
    if keys is None:                                       # graphs from the columnar constructor: rebuild the key map from the names
        keys = {(G._stem(n) if merge else n): i for i, n in enumerate(g.meta["names"])}
    key_of = (lambda p_: G._stem(p_)) if merge else (lambda p_: p_)
    evs = G.resolve_event_paths(events)                    # path-less (write) events follow the pid's open file
    t0 = G._parse_ts(evs[0]["timestamp"]) if evs else 0.0
    span = max(G._parse_ts(evs[-1]["timestamp"]) - t0, 1e-6) if evs else 1.0
    per_file: dict = {}
    for j, e in enumerate(evs):
        node = keys.get(key_of(e["path"]))
        if node is None or g.meta["node_kind"][node] != 0:
            continue
        per_file.setdefault(node, []).append((j, e))
    nodes = sorted(per_file)
    seq = np.zeros((len(nodes), t_max, lstm.D_IN), np.float32)
    lengths = np.zeros(len(nodes), np.int32)
    step_event = np.full((len(nodes), t_max), -1, np.int64)
    for i, n in enumerate(nodes):
        es = per_file[n][-t_max:]
        lengths[i] = len(es)
        prev = None
        for k, (j, e) in enumerate(es):
            step_event[i, k] = j
            t = G._parse_ts(e["timestamp"])
            slot = _SEQ_EVENT_SLOT.get(e["event"], 7)
            seq[i, k, G.OBSERVABLE_SLOT[slot] if observable else slot] = 1.0
            seq[i, k, 8] = np.log1p(float(G.clamp_bytes(e.get("size", 0)))) / 20.0
            seq[i, k, 9] = min(t - prev, 10.0) if prev is not None else 0.0
            seq[i, k, 10] = (t - t0) / span
            seq[i, k, 11] = 1.0 if ".lockbit" in e["path"] else 0.0
            seq[i, k, 12] = 1.0 if e["path"].startswith(("/tmp", "/proc")) else 0.0
            prev = t
    if return_events:
        return seq, lengths, np.asarray(nodes, np.int64), step_event
    return seq, lengths, np.asarray(nodes, np.int64)


@dataclass
class PipelineResult:
    node_score: torch.Tensor
    candidates: np.ndarray            # node id of each action (the A candidate files; kills: pid nodes; restores: -1)
    probs: torch.Tensor               # [A, 2] encrypt_probability, ransomware_score
    plan: mcts.Plan
    plan_nodes: list                  # node ids to revert, in plan order
    timings_ms: dict = field(default_factory=dict)
    n_kill: int = 0                   # the first n_kill candidates are process nodes ("kill process" actions)
    kill_attribution: str | None = None   # how files were attributed to processes: "writer" (last process in-edge) or
                                          # "edges" (the trained edge head); None when no kill actions were proposed
    n_restore: int = 0                # "restore from backup" actions proposed (state word 0, after the kills)
    restores: list = field(default_factory=list)   # per APPLIED restore, in plan order: {"position": index in plan.actions,
                                                   # "dir": directory, "dir_hash": int, "covers": covered node ids}
    actions: Actions | None = None    # the action set the plan was made over (cand[i] is the node of action i)
    evidence: dict | None = None      # run(explain=k): node id of each planned node step -> its explanation
                                      # (explain.explain_nodes + explain.attach_events); None when not asked for
    sequence_evidence: dict | None = None   # run(explain_sequences=k): node id of each planned file step -> the BiLSTM
                                            # explanation of its sequence (explain.explain_sequences); None when not asked for
    contamination: dict | None = None  # run(contamination=True): incident id -> its contaminated nodes (taint.contamination)
    incidents: list | None = None     # run(incidents=True): the window's incidents (incident.incidents), onset order
    step_incident: dict | None = None  # run(incidents=True): node id of each planned node step and of each file an applied
                                       # restore covers -> its incident id (a kill: the incident its process owns, or None)
    file_recovery: dict | None = None  # run(incidents=True): node id of each flagged file -> (onset, event record, later
                                       # events of other processes)


@dataclass
class DistContext:
    """Multi-GPU form of the pipeline (SURVEY.md 8e rows LSTM / MCTS / e2e): one process per GPU, every rank holds the
    graph; GraphSAGE-T runs 1-D edge-block sharded with the fused per-layer exchange, the own-row scores are
    all-gathered, the LSTM batch is split across ranks and all-gathered, MCTS is root-parallel (rank r searches with
    seed + r, root statistics summed in rank order) -- every rank ends with the same plan."""
    rank: int
    world: int
    exchange: str = "broadcast"      # NCCL all-gather-v per layer: window graphs change size every tick, so the peer-mapped
                                     # buffers of the fused exchange (sized by N, collectively allocated) would be rebuilt per tick


def _sage_scores(g_dev, model, ctx):
    """-> (node scores, final embeddings h); h is None on the sharded multi-GPU path."""
    x, rp, col, ew = g_dev
    if ctx is None or ctx.world == 1:
        h, score = model(x, rp, col, ew)
        return score, h
    import torch.distributed as dist
    from . import dist as ND
    ss = ND.ShardedSage(model, rp, col, ew, ctx.rank, ctx.world, x.device, exchange=ctx.exchange)
    ss.set_x(x)
    score = ss.step()
    cuts = ss.shard.cuts
    parts = [torch.empty(int(cuts[p + 1] - cuts[p]), device=x.device) for p in range(ctx.world)]
    dist.all_gather(parts, score[int(cuts[ctx.rank]):int(cuts[ctx.rank + 1])].contiguous())
    return torch.cat(parts), None


def _lstm_probs(seq_model, seq_sel, len_sel, dev, ctx):
    if torch.is_tensor(seq_sel):                                       # built on the device (stream.DeviceStream.sequences_device)
        return seq_model(seq_sel.to(dev), len_sel.to(dev))
    if ctx is None or ctx.world == 1 or seq_sel.shape[0] < ctx.world:
        return seq_model(torch.from_numpy(seq_sel).to(dev), torch.from_numpy(len_sel).to(dev))
    import torch.distributed as dist
    a = seq_sel.shape[0]
    per = (a + ctx.world - 1) // ctx.world
    lo, hi = min(ctx.rank * per, a), min((ctx.rank + 1) * per, a)
    mine = torch.zeros(per, 2, device=dev)
    if hi > lo:
        mine[:hi - lo] = seq_model(torch.from_numpy(seq_sel[lo:hi]).to(dev), torch.from_numpy(len_sel[lo:hi]).to(dev))
    parts = [torch.empty(per, 2, device=dev) for _ in range(ctx.world)]
    dist.all_gather(parts, mine)
    return torch.cat(parts)[:a]


def _edge_rows(rp: torch.Tensor, cand: torch.Tensor):
    """CSR positions of the in-edges of the rows `cand`, row by row: (edge index [m], candidate index [m])."""
    deg = (rp[cand + 1] - rp[cand]).numpy()
    seg = np.repeat(np.arange(cand.shape[0], dtype=np.int64), deg)
    start = np.cumsum(deg) - deg
    idx = np.repeat(rp[cand].numpy(), deg) + np.arange(seg.shape[0], dtype=np.int64) - np.repeat(start, deg)
    return idx, seg


def process_kill_candidates(g: G.TemporalGraph, candidates: np.ndarray, max_kills: int = 32, edge_attack=None):
    """Non-revert undo candidates derived from the graph (threat-model.mdx:208-222 "Kill process", cost 10): the
    process nodes that own the candidate files, the ones with the most candidate files first.
    A file's owner is its last writer (the source of its most recent process in-edge) -- or, given `edge_attack`
    (P(attack) [E] per CSR edge, from a trained edge head), the process source in its row with the highest P(attack),
    ties to the latest edge: a backup agent or scanner that opened an encrypted file after the ransomware is then not
    taken for its writer.
    -> (pid_nodes [k], guard [A] = index into pid_nodes of the owner of each candidate file, or -1)."""
    return _owners_to_kills(file_owners(g, candidates, edge_attack), max_kills)


def file_owners(g: G.TemporalGraph, files, edge_attack=None) -> np.ndarray:
    """The process node that owns each of `files` (int64 [len(files)], -1 when its row has no process source): the source
    of its last process in-edge (rows are time-sorted: its last writer), or, given `edge_attack` (P(attack) [E] per CSR
    edge), the process source in its row with the highest P(attack), ties to the later edge.  The attribution rule of
    process_kill_candidates and of incidents (DESIGN.md 1.4)."""
    kind = torch.as_tensor(np.asarray(g.meta["node_kind"]))
    rp = (g.rowptr.cpu() if torch.is_tensor(g.rowptr) else torch.from_numpy(np.asarray(g.rowptr))).long()
    col = (g.col.cpu() if torch.is_tensor(g.col) else torch.from_numpy(np.asarray(g.col))).long()
    cand = torch.from_numpy(np.asarray(files, np.int64))
    if edge_attack is not None:
        ea = edge_attack.detach().cpu().numpy() if torch.is_tensor(edge_attack) else edge_attack
        return _edge_owners(kind, rp, col, cand, np.asarray(ea, np.float32))
    # the most recent in-edge of a file node (rows are time-sorted) whose source is a process = its last writer
    owner = np.full(cand.shape[0], -1, np.int64)
    last = rp[cand + 1] - 1
    has = (rp[cand + 1] > rp[cand]).numpy()
    src = col[last.clamp_min(0)]
    is_proc = (kind[src] == 1).numpy() & has
    owner[is_proc] = src.numpy()[is_proc]
    for i in np.nonzero(has & ~is_proc)[0].tolist():          # rare: the last toucher is a file (rename link): scan back
        n = int(cand[i]); s_ = col[rp[n]:rp[n + 1]]; s_ = s_[kind[s_] == 1]
        if s_.numel():
            owner[i] = int(s_[-1])
    return owner


def _owners_to_kills(owner: np.ndarray, max_kills: int):
    pids, counts = np.unique(owner[owner >= 0], return_counts=True)
    if pids.size == 0:
        return np.zeros(0, np.int64), np.full(owner.shape[0], -1, np.int64)
    chosen = pids[np.lexsort((pids, -counts))[:max_kills]]
    slot = np.full(int(max(pids.max(), 0)) + 1, -1, np.int64); slot[chosen] = np.arange(chosen.shape[0])
    guard = np.where(owner >= 0, slot[np.maximum(owner, 0)], -1)
    return chosen, guard


def _edge_owners(kind, rp, col, cand, edge_attack):
    """Per candidate file: the process source of its row with the highest P(attack), ties to the latest edge; -1 if none."""
    idx, seg = _edge_rows(rp, cand)
    src = col.numpy()[idx]
    keep = kind.numpy()[src] == 1
    idx, seg, src = idx[keep], seg[keep], src[keep]
    owner = np.full(cand.shape[0], -1, np.int64)
    if idx.size:
        o = np.lexsort((idx, edge_attack[idx], seg))           # per row ascending (P(attack), position): the last one wins
        last = np.ones(o.shape[0], bool); last[:-1] = seg[o][1:] != seg[o][:-1]
        owner[seg[o][last]] = src[o][last]
    return owner


def edge_kill_confidence(g: G.TemporalGraph, candidates: np.ndarray, pids: np.ndarray, edge_attack) -> np.ndarray:
    """Confidence that each process in `pids` is malicious: the highest P(attack) over its edges into the candidate
    files (0 if it has none)."""
    rp = (g.rowptr.cpu() if torch.is_tensor(g.rowptr) else torch.from_numpy(np.asarray(g.rowptr))).long()
    col = (g.col.cpu() if torch.is_tensor(g.col) else torch.from_numpy(np.asarray(g.col))).long()
    idx, _ = _edge_rows(rp, torch.from_numpy(np.asarray(candidates, np.int64)))
    src = col.numpy()[idx]
    ea = np.asarray(edge_attack, np.float32)[idx]
    out = np.zeros(len(pids), np.float32)
    for k, p_ in enumerate(np.asarray(pids).tolist()):
        m = src == p_
        if m.any():
            out[k] = ea[m].max()
    return out


def node_dir_hashes(g: G.TemporalGraph, nodes=None):
    """int64 parent-directory hash (stream.dir_hash) of the given nodes (all when None): on the device for graphs of a
    device-resident stream (nerrf_trace_dir_hash_ex), from the name strings and meta["node_source"] for host graphs --
    qualified by each node's source either way, so a directory group never spans two hosts."""
    from .stream import dir_hash
    fn = g.meta.get("dir_hash")
    if callable(fn):
        dh = fn()
        return dh if nodes is None else dh[torch.as_tensor(np.asarray(nodes, np.int64)).to(dh.device)]
    names = g.meta["names"]
    src = g.meta.get("node_source")
    idx = range(len(names)) if nodes is None else np.asarray(nodes, np.int64).tolist()
    return torch.tensor([dir_hash(names[int(i)], 0 if src is None else int(src[int(i)])) for i in idx], dtype=torch.int64)


def propose_restores(cand_dir, file_dir, file_size, file_is_cand, max_restores: int = 4, min_files: int = 8):
    """"Restore from backup" candidates (threat-model.mdx:216-219, cost 100): the directories holding the most candidate
    files (at least `min_files`), at most `max_restores`, most candidates first (ties: lower hash).
    cand_dir int64 [A]: directory hash of each candidate file; file_dir / file_size / file_is_cand [F]: every file node of
    the window.  A restore's collateral is the summed size of the directory's files that are NOT candidates: it assumes
    the snapshot clobbers every other file the window saw there (conservative).
    -> (dir hashes int64 [k], collateral fp32 [k], slot of each candidate int64 [A]: index into the k restores or -1)."""
    cand_dir = torch.as_tensor(cand_dir).cpu()
    dirs, counts = torch.unique(cand_dir, return_counts=True)
    ok = counts >= min_files
    dirs, counts = dirs[ok].numpy(), counts[ok].numpy()
    chosen = dirs[np.lexsort((dirs, -counts))[:max_restores]]
    slot = np.full(cand_dir.shape[0], -1, np.int64)
    if chosen.size == 0:
        return chosen, np.zeros(0, np.float32), slot
    slot_of = {int(d): k for k, d in enumerate(chosen.tolist())}
    slot = np.array([slot_of.get(int(d), -1) for d in cand_dir.tolist()], np.int64)
    file_dir = torch.as_tensor(file_dir)
    ch = torch.from_numpy(chosen).to(file_dir.device)
    other = ~torch.as_tensor(file_is_cand).to(file_dir.device)
    size = torch.as_tensor(file_size).to(file_dir.device).to(torch.float64)
    coll = np.zeros(chosen.shape[0], np.float64)
    hit = other & torch.isin(file_dir, ch)
    if bool(hit.any()):
        d_hit, s_hit = file_dir[hit].cpu().numpy(), size[hit].cpu().numpy()
        for k, d in enumerate(chosen.tolist()):
            coll[k] = s_hit[d_hit == d].sum()
    return chosen, coll.astype(np.float32), slot


def run(g: G.TemporalGraph, seq, lengths, seq_nodes, model: GraphSAGE_T, seq_model, top_a=1024, confidence=None,
        plan_steps=None, n_rollouts=4096, depth=50, iterations=16, device="cuda", exclude=None, commit_per_search=1,
        dist_ctx: DistContext | None = None, kill_candidates: bool = False, restore_candidates: bool = False,
        max_restores: int = 4, min_restore_files: int = 8, explain: int = 0,
        explain_max_edges: int | None = None, explain_max_full_graph: int | None = None, explain_sequences: int = 0,
        seq_events=None, incidents: bool = False, incident_tau: float = 0.5, host_names=None, contamination: bool = False,
        contamination_hops: int = -1, contamination_only=None) -> PipelineResult:
    """seq/lengths/seq_nodes: LSTM inputs for (a superset of) the candidate file nodes (file_sequences()).
    seq may instead be a CALLABLE nodes -> (seq, lengths, nodes_with_sequences): the sequences are then built only for
    the top-A candidates (large windows: a million file nodes, a few thousand candidates); seq_nodes = the file nodes.
    confidence: optional override of p_a per NODE (e.g. ground-truth labels when no trained weights exist).
    exclude: bool [len(seq_nodes)] -- sequences whose file was already reverted by an earlier tick of the stream.
    kill_candidates: also propose "kill process" actions (cost 10) for the processes that wrote the candidate files;
    a file reversion only sticks once its writer is gone (planner spec v1, DESIGN.md 1.3).  A model marked
    `edge_head_trained` (ai.train with edge_weight > 0) attributes files to processes by its edge head instead of the
    last-writer rule, on one GPU; res.kill_attribution records which rule ran.
    restore_candidates: also propose "restore from backup" actions (cost 100) for the (at most `max_restores`) parent
    directories holding the most candidate files (at least `min_restore_files`); a restore covers every candidate file of
    its directory and costs the directory's other files as collateral (planner spec v2, DESIGN.md 1.3).  Restores take
    the state-word-0 slots after the kills (kill budget 32 - restores).  res.plan_nodes lists node actions only;
    res.restores lists the applied restores.
    explain = k > 0: after planning, res.evidence holds each planned node's k strongest GraphSAGE-T edge attributions with
    their events (nerrf_b200.explain; a kill step explains its process node, restores carry none).  The plan is the
    plan of explain=0.  One GPU only.
    explain_sequences = k > 0: res.sequence_evidence holds, for each planned file step, the k steps of its event sequence
    that drove the BiLSTM's encrypt logit most (explain.explain_sequences), with their events; kills and restores carry
    none.  seq_events: the event of each step of `seq` (int64 [len(seq), T], file_sequences(return_events=True)); a
    callable `seq` is then called as seq(nodes, events=True) and returns a fourth value, the same for its sequences.
    Events of both kinds of evidence are resolved in one g.meta["event_info"] call.  The plan is the plan of
    explain_sequences=0.  One GPU only.
    incidents=True: res.incidents holds the window's incidents (DESIGN.md 1.4; incident.incidents over the files scored
    >= incident_tau plus the plan's file steps and the files its applied restores cover, so every file step has one),
    res.step_incident each planned node step's incident id and res.file_recovery each flagged file's recovery point.
    Files are attributed by the edge head exactly when the kill attribution is (a model marked edge_head_trained).
    host_names: source id -> host name, the prefix of incident ids on a graph of several sources.  The plan is the plan
    of incidents=False.  One GPU only.
    contamination=True (needs incidents=True): res.contamination holds what each incident's attack spread to (DESIGN.md
    1.5; taint.contamination over at most contamination_hops hops, -1 = unbounded; contamination_only=ID seeds that
    incident alone).  The plan is the plan of contamination=False.  One GPU only."""
    if contamination and not incidents:
        raise ValueError("contamination=True needs incidents=True (the closure is seeded by the incidents)")
    if contamination and dist_ctx is not None and dist_ctx.world > 1:
        raise NotImplementedError("contamination is computed on one GPU (dist_ctx.world > 1 is not supported)")
    if incidents and dist_ctx is not None and dist_ctx.world > 1:
        raise NotImplementedError("incidents are computed on one GPU (dist_ctx.world > 1 is not supported)")
    if restore_candidates and dist_ctx is not None and dist_ctx.world > 1:
        raise NotImplementedError("restore candidates are planned on one GPU (dist_ctx.world > 1 is not supported)")
    if (explain or explain_sequences) and dist_ctx is not None and dist_ctx.world > 1:
        raise NotImplementedError("explanations are computed on one GPU (dist_ctx.world > 1 is not supported)")
    dev = torch.device(device)
    tm = {}
    sync = torch.cuda.synchronize

    t0 = time.perf_counter()
    # numpy arrays (host constructor) are uploaded; CUDA tensors (ingest.graph_from_columns(device=...)) are used as is
    x, rp, col, ew = ((a if torch.is_tensor(a) else torch.from_numpy(a)).to(dev, non_blocking=True)
                      for a in (g.x, g.rowptr, g.col, g.ew))
    sync(); tm["h2d_graph"] = (time.perf_counter() - t0) * 1e3

    t0 = time.perf_counter()
    score, h_final = _sage_scores((x, rp, col, ew), model, dist_ctx)
    sync(); tm["graphsage_t"] = (time.perf_counter() - t0) * 1e3

    t0 = time.perf_counter()
    seq_nodes_t = torch.from_numpy(np.asarray(seq_nodes)).to(dev)
    cand_score = score[seq_nodes_t]
    if exclude is not None and np.asarray(exclude).any():
        cand_score = cand_score.masked_fill(torch.from_numpy(np.asarray(exclude)).to(dev), -1.0)
    a = min(top_a, int(seq_nodes_t.numel() if exclude is None else (~np.asarray(exclude)).sum()))
    if a == 0:
        return PipelineResult(score, np.zeros(0, np.int64), torch.zeros(0, 2, device=dev), mcts.Plan([], [0.0], []), [], dict(tm, total=sum(tm.values())))
    cand_local = torch.topk(cand_score, a).indices                   # most anomalous files that have sequences
    candidates = seq_nodes_t[cand_local]
    sync(); tm["top_a"] = (time.perf_counter() - t0) * 1e3

    t0 = time.perf_counter()
    ev_sel = None
    if callable(seq):
        want = candidates.cpu().numpy()
        if explain_sequences:
            sq, ln, have, ev = seq(want, events=True)                  # ... and the event of every step
        else:
            sq, ln, have = seq(want)                                   # sequences of the candidates only
        if have is None:                                               # already in candidate order (device builder: CUDA tensors)
            seq_sel, len_sel = sq, ln
            ev_sel = ev if explain_sequences else None
        else:                                                          # sorted by node id (host builder)
            pos = np.searchsorted(have, want)
            assert have.shape[0] == want.shape[0] and np.array_equal(have[pos], want), "every candidate file has events"
            seq_sel, len_sel = sq[pos], ln[pos]
            ev_sel = ev[pos] if explain_sequences else None
        tm["sequences"] = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
    else:
        cl = cand_local.cpu().numpy()
        seq_sel, len_sel = seq[cl], lengths[cl]
        if explain_sequences and seq_events is not None:
            ev_sel = np.asarray(seq_events)[cl]
    probs = _lstm_probs(seq_model, seq_sel, len_sel, dev, dist_ctx)
    sync(); tm["lstm"] = (time.perf_counter() - t0) * 1e3

    t0 = time.perf_counter()
    cand = candidates.cpu().numpy()
    size_all_nodes = g.meta.get("size_mb", np.ones(g.num_nodes, np.float32))
    size_mb = np.maximum(size_all_nodes[cand], 0.01)
    n_kill = 0
    r_dirs, r_slot = np.zeros(0, np.int64), None
    if restore_candidates:
        files = np.nonzero(np.asarray(g.meta["node_kind"]) == 0)[0]
        file_dir = node_dir_hashes(g, files)
        is_cand = torch.from_numpy(np.isin(files, cand))
        r_dirs, r_coll, r_slot = propose_restores(node_dir_hashes(g, cand), file_dir, np.asarray(size_all_nodes, np.float32)[files],
                                                  is_cand, min(max_restores, 32), min_restore_files)
    n_restore = int(r_dirs.shape[0])
    edge_attack = None                                                 # P(attack) per CSR edge when the edge head attributes
    if confidence is not None:
        p = np.asarray(confidence, np.float32)[cand]
        actions = Actions(p, size_mb, np.ones(a, np.float32))
    elif kill_candidates:
        if getattr(model, "edge_head_trained", False) and h_final is not None and model.edge_W is not None:
            # files are attributed to processes by the trained edge head (P(attack) of each CSR edge)
            _, el = model.heads(h_final, rp, col, return_edge_logits=True)
            edge_attack = torch.softmax(el, 1)[:, 0].cpu().numpy()
        pids, guard = process_kill_candidates(g, cand, max_kills=32 - n_restore, edge_attack=edge_attack)
        n_kill = int(pids.shape[0])
        a_rev = min(a, 4096 - n_kill - n_restore)                      # kill actions occupy the first slots (spec v1: guards < 32)
        p_rev = 0.5 * (score[candidates[:a_rev]].cpu().numpy() + probs[:a_rev, 0].cpu().numpy())
        gr = guard[:a_rev]
        if edge_attack is not None:
            # confidence that a process is malicious = the highest P(attack) over its edges into the candidate files
            p_kill = edge_kill_confidence(g, cand, pids, edge_attack)
        else:
            # confidence that a process is malicious = mean confidence of the candidate files it wrote (the model's node
            # head is trained on file nodes only)
            p_kill = np.array([p_rev[gr == k].mean() if (gr == k).any() else 0.0 for k in range(n_kill)], np.float32)
        p_all = np.concatenate([p_kill, p_rev]).astype(np.float32)
        size_all = np.concatenate([np.zeros(n_kill, np.float32), size_mb[:a_rev]])
        kind = np.concatenate([np.full(n_kill, RW_KIND_KILL, np.int64), np.zeros(a_rev, np.int64)])
        cost = np.where(kind == RW_KIND_KILL, 10.0, 1.0).astype(np.float32)
        actions = Actions(p_all, size_all, cost, kind, guard=np.concatenate([np.full(n_kill, -1, np.int64), guard[:a_rev]]))
        cand = np.concatenate([pids, cand[:a_rev]])
    else:
        actions = Actions.from_scores(score[candidates], probs[:, 0], size_mb, np.zeros(a, np.int64))
    if n_restore:
        # restore actions take the word-0 slots after the kills: p = 0, size = collateral (u = 0, v = collateral), cost 100;
        # every candidate file of a restored directory names its restore as its cover.  Kill (guard) slots stay below nk.
        nk = n_kill
        a_rev = min(actions.A - nk, 4096 - nk - n_restore)
        ins = lambda x, mid: np.concatenate([x[:nk], mid, x[nk:nk + a_rev]])
        kind = actions.kind if actions.kind is not None else np.zeros(actions.A, np.int64)
        guard = actions.guard if actions.guard is not None else np.full(actions.A, -1, np.int32)
        cover = np.where(r_slot[:a_rev] >= 0, nk + r_slot[:a_rev], -1)
        actions = Actions(ins(actions.p, np.zeros(n_restore, np.float32)), ins(actions.size, r_coll),
                          ins(actions.cost, np.full(n_restore, KIND_COST[RW_KIND_RESTORE], np.float32)),
                          ins(kind, np.full(n_restore, RW_KIND_RESTORE, np.int64)),
                          guard=ins(guard, np.full(n_restore, -1, np.int32)),
                          cover=np.concatenate([np.full(nk + n_restore, -1, np.int64), cover]))
        cand = ins(cand, np.full(n_restore, -1, np.int64))
    merge = None
    if dist_ctx is not None and dist_ctx.world > 1:
        from . import dist as ND
        merge = lambda n, w: ND.root_parallel_search(lambda off: (n, w), dist_ctx.rank, dist_ctx.world)
    pl = mcts.plan(actions, max_steps=plan_steps, n_rollouts=n_rollouts, depth=depth, seed=dist_ctx.rank if dist_ctx else 0,
                   iterations=iterations, device=dev, commit_per_search=commit_per_search, merge=merge)
    sync(); tm["mcts_plan"] = (time.perf_counter() - t0) * 1e3
    tm["total"] = sum(tm.values())
    is_restore = lambda i: n_kill <= i < n_kill + n_restore
    res = PipelineResult(score, cand, probs, pl, [int(cand[i]) for i in pl.actions if not is_restore(i)], tm)
    res.n_kill = n_kill
    res.n_restore = n_restore
    res.actions = actions
    if n_restore:
        names = g.meta.get("names")
        for k, i in enumerate(pl.actions):
            if is_restore(i):
                covers = cand[np.nonzero(actions.cover == i)[0]].tolist() if actions.cover is not None else []
                d = ""
                if names is not None and covers:
                    from .stream import parent_dir
                    d = parent_dir(names.take([covers[0]])[0] if hasattr(names, "take") else names[covers[0]])
                res.restores.append({"position": k, "dir": d, "dir_hash": int(r_dirs[i - n_kill]), "covers": [int(c) for c in covers]})
    if confidence is None and kill_candidates:
        res.kill_attribution = "writer" if edge_attack is None else "edges"
    if incidents:
        tm["incidents"] = _label_incidents(res, g, (rp, col, ew, x), model, h_final, score, incident_tau, host_names,
                                           edge_attack)
        if contamination:
            t0 = time.perf_counter()
            res.contamination = contamination_of(G.TemporalGraph(rp, col, ew, x, g.meta), res, contamination_hops,
                                                 contamination_only)
            tm["contamination"] = (time.perf_counter() - t0) * 1e3
    if explain or explain_sequences:
        from . import explain as X
        t0 = time.perf_counter()
        todo = list(dict.fromkeys(res.plan_nodes))
        ex = []
        if explain:
            kw = {}
            if explain_max_edges is not None:
                kw["max_edges_per_target"] = explain_max_edges
            if explain_max_full_graph is not None:
                kw["max_full_graph_targets"] = explain_max_full_graph
            ex = X.explain_nodes(G.TemporalGraph(rp, col, ew, x, g.meta), model, todo, k=int(explain), **kw)
            sync()
        t1 = time.perf_counter()
        files, sx = [], None
        if explain_sequences:
            row = {int(c): j for j, c in enumerate(candidates.cpu().numpy().tolist())}   # a file step's row of seq_sel
            files = [n for n in todo if n in row]
            idx = np.asarray([row[n] for n in files], np.int64)
            take = lambda a: a[torch.from_numpy(idx).to(a.device)] if torch.is_tensor(a) else np.asarray(a)[idx]
            sx = X.explain_sequences(seq_model, take(seq_sel), take(len_sel), k=int(explain_sequences),
                                     step_event=None if ev_sel is None else take(ev_sel))
            sync()
        t2 = time.perf_counter()
        if sx is None:
            ex = X.attach_events(g, ex)
        else:
            ex, sx = X.attach_events(g, ex, sx)                        # one event_info call for both kinds of evidence
            res.sequence_evidence = dict(zip(files, sx))
        if explain:
            res.evidence = dict(zip(todo, ex))
        t3 = time.perf_counter()
        if explain:
            tm["explain"] = (t1 - t0 + t3 - t2) * 1e3
        if explain_sequences:
            tm["explain_sequences"] = (t2 - t1 + (0.0 if explain else t3 - t2)) * 1e3
    return res


def _label_incidents(res: PipelineResult, g, g_dev, model, h_final, score, tau, host_names, edge_attack=None):
    """fill res.incidents / step_incident / file_recovery (run(incidents=True)) -> the time it took (ms).  edge_attack: the
    P(attack) the kill attribution used, if it ran; otherwise the edge head's is computed here when the model has one."""
    from . import incident as I
    rp, col, ew, x = g_dev
    t0 = time.perf_counter()
    kind = np.asarray(g.meta["node_kind"])
    seeds = [n for n in res.plan_nodes if kind[n] == 0] + [c for r in res.restores for c in r["covers"]]
    if edge_attack is None and getattr(model, "edge_head_trained", False) and h_final is not None and model.edge_W is not None:
        _, el = model.heads(h_final, rp, col, return_edge_logits=True)
        edge_attack = torch.softmax(el, 1)[:, 0].contiguous()
    recs, per_file = I.incidents(G.TemporalGraph(rp, col, ew, x, g.meta), score, tau=tau, seeds=np.unique(np.asarray(seeds, np.int64)),
                                 edge_attack=edge_attack, host_names=host_names, return_files=True)
    res.incidents = recs
    res.step_incident = step_incidents(res.plan_nodes, res.restores, kind, recs, per_file)
    res.file_recovery = {v: (f["onset"], f["event"], f["later"]) for v, f in per_file.items()}
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def contamination_of(g, res: PipelineResult, max_hops=-1, only=None, device="cuda") -> dict:
    """taint.contamination seeded by a run(incidents=True) result: its incidents, and each flagged file at its recovery
    point (res.file_recovery).  `g` is uploaded to `device` when its arrays are on the host."""
    from . import taint
    if not torch.is_tensor(g.rowptr):
        dev = torch.device(device)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        g = G.TemporalGraph(up(g.rowptr), up(g.col), up(g.ew), up(g.x), g.meta)
    per_file = {int(v): {"onset": r[0]} for v, r in (res.file_recovery or {}).items()}
    return taint.contamination(g, res.incidents or [], per_file, max_hops=max_hops, only=only)


def step_incidents(plan_nodes, restores, node_kind, recs, per_file) -> dict:
    """node id -> incident id, for every planned node step (a file: its own incident; a kill: the incident whose owner is
    the killed process, or None) and every file an applied restore covers (covered files are not plan nodes: the emitter
    labels a restore with its covers' incidents)"""
    by_owner = {r["owner"]: r["id"] for r in recs if r["owner"] >= 0}
    out = {int(n): (per_file[int(n)]["incident"] if node_kind[n] == 0 else by_owner.get(int(n))) for n in plan_nodes}
    for r in restores:
        for c in r["covers"]:
            out[int(c)] = per_file[int(c)]["incident"]
    return out
