"""Undo-plan emitter: the step AFTER the hot path (SURVEY.md 8f rank 4) -- host code only.

Turns a planner result (ordered action indices over candidate file nodes) into the artefact the
reference hands to its sandbox / `nerrf undo` CLI: an ordered list of file reversions with the
validation rule the sandbox applies.

Reference anchors (prose + the M1 harness; no emitter exists in the reference):
  * planner output "Undo plan (file reversions, process kills)"  docs/content/docs/architecture.mdx:62-72
  * sandbox workflow "apply undo operations ... validate: md5sum matches pre-attack version ...
    approve if all checks pass"                                    docs/content/docs/architecture.mdx:75-86
  * what a reversion IS for the LockBit simulator: `x.lockbit3` -> `x.dat`
                                                                   benchmarks/m1/scripts/m1_rollback.sh:95-112
  * CLI `nerrf undo --id <attack>`                                 ROADMAP.md:28,86
[ours]: the JSON field names (the reference defines none); version field so they can change.
"""
from __future__ import annotations

import json
import re
import shlex

import numpy as np

PLAN_VERSION = 1
ENCRYPTED_SUFFIX = ".lockbit3"      # benchmarks/m1/scripts/m1_rollback.sh:95 (`for f in *.lockbit3`)
RESTORED_SUFFIX = ".dat"            # benchmarks/m1/scripts/m1_rollback.sh:98 (`mv "$f" "${base}.dat"`)


_HOST_NAME = re.compile(r"[A-Za-z0-9._-]{1,64}")


def check_host_name(name) -> str:
    """A source (host) name becomes a file name (<host>.sh) and a plan field: 1-64 characters of [A-Za-z0-9._-], and
    not "." or ".." (which name directories).  Anything else raises ValueError."""
    if not isinstance(name, str) or not _HOST_NAME.fullmatch(name) or name in (".", ".."):
        raise ValueError("bad host name %r: 1-64 characters of [A-Za-z0-9._-], not '.' or '..'" % (name,))
    return name


def _has_control_chars(path: str) -> bool:
    return any(ord(ch) < 0x20 or ord(ch) == 0x7F for ch in path)


def reversion_for(path: str) -> dict:
    """One file reversion.  An encrypted twin is renamed back (the M1 harness' recovery); anything else
    has no in-place inverse and is restored from the pre-attack snapshot the sandbox cloned.
    Paths come from attacker-controlled file names in the trace: an empty path is refused (it names no file;
    the tracker zeroes `path` on write events, tracker/bpf/tracepoints.c:62-64), and a path with control
    characters is flagged so that no consumer ever pastes it into a line-oriented format."""
    if not path:
        raise ValueError("cannot emit a reversion for an empty path")
    if path.endswith(ENCRYPTED_SUFFIX):
        r = {"op": "rename", "from": path, "to": path[: -len(ENCRYPTED_SUFFIX)] + RESTORED_SUFFIX}
    else:
        r = {"op": "restore_snapshot", "path": path}
    if _has_control_chars(path):
        r["hostile_name"] = True       # exact bytes kept (JSON escapes them); to_shell() only ever passes them as a quoted argument
    return r


def restore_dir_step(directory: str, covered_paths) -> dict:
    """One directory restore from the pre-attack snapshot (threat-model.mdx:216-219 "Restore from backup"): brings back
    every file of `directory`; the sandbox checks each covered file against its pre-attack md5."""
    r = {"op": "restore_snapshot_dir", "dir": directory, "covers": list(covered_paths),
         "validate": [{"check": "md5", "path": p_, "against": "pre_attack_snapshot"} for p_ in covered_paths]}
    if _has_control_chars(directory) or any(_has_control_chars(p_) for p_ in covered_paths):
        r["hostile_name"] = True
    return r


def event_fields(ev, host_names=None):
    """The plan record of one evidence event (an event_info record, or None) -> (record or None, hostile): record =
    {"time", "pid", "syscall", "path"[, "host"]}; hostile = a control character in its path or syscall."""
    if ev is None:
        return None, False
    rec = {"time": float(ev["time"]), "pid": int(ev["pid"]), "syscall": str(ev["syscall"]), "path": str(ev["path"])}
    if host_names is not None and "source" in ev:
        rec["host"] = check_host_name(host_names[int(ev["source"])])
    return rec, _has_control_chars(rec["path"]) or _has_control_chars(rec["syscall"])


def sequence_evidence_fields(sx, host_names=None) -> dict:
    """The plan fields of one file's sequence explanation (pipeline.PipelineResult.sequence_evidence[node]):
    "sequence_evidence" = one entry per attributed step, strongest first -- {"event": {"time", "pid", "syscall",
    "path"[, "host"]}, "step" (position in the file's sequence, oldest first), "feature" (name of the step's dominant
    feature, lstm.FEATURE_NAMES; None when every term is 0), "attribution"} -- and "sequence_evidence_logit" (the
    BiLSTM's encrypt logit).  A control character in an event's path flags the step "hostile_name"."""
    from ..models.lstm import FEATURE_NAMES
    out, hostile = [], False
    for s in sx["steps"]:
        rec, bad = event_fields(s.get("event"), host_names)
        hostile = hostile or bad
        f = int(s["feature"])
        out.append({"event": rec, "step": int(s["t"]), "feature": FEATURE_NAMES[f] if 0 <= f < len(FEATURE_NAMES) else None,
                    "attribution": float(s["attr"])})
    r = {"sequence_evidence": out, "sequence_evidence_logit": float(sx["logit"])}
    if hostile:
        r["hostile_name"] = True
    return r


def evidence_fields(ex, host_names=None) -> dict:
    """The plan fields of one node's explanation (pipeline.PipelineResult.evidence[node]): "evidence" = one entry per
    attributed edge, strongest first -- {"event": {"time", "pid", "syscall", "path"[, "host"]}, "src", "dst" (the edge's
    two node names), "attribution"} -- and "evidence_logit"; or "evidence": None with "evidence_reason" when the node
    was not explained.  host_names: source id -> host name (several sources).  Names and paths come from the trace:
    a control character in any of them flags the step "hostile_name", as for the step's own path."""
    if ex.get("scope") is None:
        return {"evidence": None, "evidence_reason": str(ex.get("reason", ""))}
    out, hostile = [], False
    for e in ex["edges"]:
        rec, bad = event_fields(e.get("event"), host_names)
        hostile = hostile or bad
        src, dst = str(e.get("src_name", e["src"])), str(e.get("dst_name", e["dst"]))
        hostile = hostile or _has_control_chars(src) or _has_control_chars(dst)
        out.append({"event": rec, "src": src, "dst": dst, "attribution": float(e["attr"])})
    r = {"evidence": out, "evidence_logit": float(ex["logit"])}
    if hostile:
        r["hostile_name"] = True
    return r


def incident_fields(inc, host_names=None) -> dict:
    """The plan record of one incident (incident.incidents): {"id", "host", "process", "files" (node ids), "n_files",
    "onset" / "end": {"time", "event"}, "size_mb", "later_other_events", "max_score"}; "hostile_name" when an event's
    path or syscall holds a control character."""
    hostile = False
    r = {"id": str(inc["id"]), "host": None if inc.get("host") is None else check_host_name(inc["host"]),
         "process": inc.get("process"), "files": [int(v) for v in inc["files"]], "n_files": int(inc["n_files"])}
    for k in ("onset", "end"):
        rec, bad = event_fields(inc.get(k + "_event"), host_names)
        hostile = hostile or bad
        r[k] = {"time": inc.get(k), "event": rec}
    r.update(size_mb=float(inc["size_mb"]), later_other_events=int(inc["later_other_events"]), max_score=inc.get("max_score"))
    if hostile:
        r["hostile_name"] = True
    return r


def contaminated_fields(c, host_names=None) -> dict:
    """The plan record of one contaminated node (taint.contamination): {"node", "name", "kind", "since", "since_event",
    "hops", "via" (the events that carried the taint to it, oldest first)}; a file also gets "recovery_point":
    {"before": since, "event": since_event} (restoring it to before the event that tainted it).  "hostile_name" when its
    name or any event's path or syscall holds a control character."""
    ev, hostile = event_fields(c.get("since_event"), host_names)
    via = []
    for e in c.get("via", []):
        rec, bad = event_fields(e, host_names)
        hostile = hostile or bad
        via.append(rec)
    name = None if c.get("name") is None else str(c["name"])
    hostile = hostile or (name is not None and _has_control_chars(name))
    r = {"node": int(c["node"]), "name": name, "kind": str(c["kind"]), "since": float(c["since"]), "since_event": ev,
         "hops": int(c["hops"]), "via": via}
    if r["kind"] == "file":
        r["recovery_point"] = {"before": r["since"], "event": ev}
    if hostile:
        r["hostile_name"] = True
    return r


def recovery_point(rec, host_names=None):
    """A file's recovery point (pipeline.PipelineResult.file_recovery[node] = (onset, event, later)) -> (the plan field
    {"before": onset, "event", "later_other_events"}, hostile)"""
    onset, ev, later = rec
    e, bad = event_fields(ev, host_names)
    return {"before": onset, "event": e, "later_other_events": int(later)}, bad


def undo_plan(names, plan_nodes, scores=None, attack_id=None, size_mb=None, node_score=None, truncated=False,
              remaining_candidates=0, restores=None, hosts=None, evidence=None, host_names=None,
              sequence_evidence=None, incidents=None, step_incident=None, file_recovery=None, contamination=None) -> dict:
    """names: node id -> path (TemporalGraph.meta['names']); plan_nodes: node ids to revert, in plan order
    (PipelineResult.plan_nodes); scores: Plan.scores (exact reward after each commit, scores[0] = before).
    truncated / remaining_candidates: the planner stopped at its step limit while improving candidates remained --
    such a plan must not be auto-approved as complete.
    restores: PipelineResult.restores -- directory restores, each at its position in the plan ({"position", "dir",
    "covers": node ids}); the node steps fill the other positions in order.
    hosts: node id -> host name, for a graph of several sources: every step gets the "host" it applies to (a restore:
    the host of the files it covers; covers on two hosts raise ValueError).  None: no host fields (one source).
    evidence: node id -> explanation (pipeline.PipelineResult.evidence): each node step found there gets the fields of
    evidence_fields (host_names: source id -> host name for its events).  None: no evidence fields.
    sequence_evidence: node id -> sequence explanation (pipeline.PipelineResult.sequence_evidence): each file step found
    there gets the fields of sequence_evidence_fields.  None: no sequence evidence fields.
    incidents / step_incident / file_recovery (pipeline.PipelineResult, run(incidents=True)): a top-level "incidents"
    table (incident_fields), "incident" (id or None) on every node step, "incidents" (the ids of its covers) on a restore,
    and "recovery_point" (recovery_point) on every file step found in file_recovery; a restore's is its earliest cover's
    point (ties to the lower node id) with later_other_events summed over the covers.  None: none of these fields.
    contamination: incident id -> contaminated nodes (pipeline.PipelineResult.contamination): each incident of the table
    gets "contaminated" (contaminated_fields, [] when it reached nothing).  None: no such field.
    to_shell reads none of the evidence or incident fields."""
    host_of = (lambda n: check_host_name(hosts[int(n)])) if hosts is not None else None
    at = {int(r["position"]): r for r in (restores or [])}
    total = len(plan_nodes) + len(at)
    nodes = iter(plan_nodes)
    steps = []
    for k in range(total):
        if k in at:
            r = at[k]
            step = {"order": k, **restore_dir_step(r["dir"], [names[int(c)] for c in r["covers"]])}
            if host_of is not None and r["covers"]:
                on = sorted({host_of(c) for c in r["covers"]})
                if len(on) > 1:
                    raise ValueError("restore of %r covers files on several hosts: %s" % (r["dir"], ", ".join(on)))
                step["host"] = on[0]
            if scores is not None and k + 1 < len(scores):
                step["reward_after"] = float(scores[k + 1])
            if step_incident is not None:
                step["incidents"] = sorted({step_incident.get(int(c)) for c in r["covers"]} - {None})
            if file_recovery is not None:
                pts = sorted((file_recovery[int(c)][0], int(c)) for c in r["covers"]
                             if int(c) in file_recovery and file_recovery[int(c)][0] is not None)
                if pts:
                    onset, ev, _ = file_recovery[pts[0][1]]
                    later = sum(int(file_recovery[int(c)][2]) for c in r["covers"] if int(c) in file_recovery)
                    rp_, bad = recovery_point((onset, ev, later), host_names)
                    step["recovery_point"] = rp_
                    if bad:
                        step["hostile_name"] = True
            steps.append(step)
            continue
        n = int(next(nodes))
        step = {"order": k, "node": n, **reversion_for(names[n]),
                "validate": {"check": "md5", "against": "pre_attack_snapshot"}}
        if host_of is not None:
            step["host"] = host_of(n)
        if size_mb is not None:
            step["size_mb"] = float(size_mb[n])
        if node_score is not None:
            step["anomaly_score"] = float(node_score[n])
        if scores is not None and k + 1 < len(scores):
            step["reward_after"] = float(scores[k + 1])
        if evidence is not None and evidence.get(n) is not None:
            step.update(evidence_fields(evidence[n], host_names))
        if sequence_evidence is not None and sequence_evidence.get(n) is not None:
            sf = sequence_evidence_fields(sequence_evidence[n], host_names)
            if sf.pop("hostile_name", False):
                step["hostile_name"] = True
            step.update(sf)
        if step_incident is not None:
            step["incident"] = step_incident.get(n)
        if file_recovery is not None and n in file_recovery:
            rp_, bad = recovery_point(file_recovery[n], host_names)
            step["recovery_point"] = rp_
            if bad:
                step["hostile_name"] = True
        steps.append(step)
    out = {"version": PLAN_VERSION, "kind": "nerrf.undo_plan", "attack_id": attack_id, "steps": steps,
           "approve_if": "all_checks_pass" if not truncated else "all_checks_pass_and_operator_confirms_partial_plan",
           "truncated": bool(truncated), "remaining_candidates": int(remaining_candidates)}
    if incidents is not None:
        out["incidents"] = [incident_fields(i, host_names) for i in incidents]
        if contamination is not None:
            for rec in out["incidents"]:
                rec["contaminated"] = [contaminated_fields(c, host_names) for c in contamination.get(rec["id"], [])]
    if scores:
        out["reward_before"] = float(scores[0])
        out["reward_after"] = float(scores[min(total, len(scores) - 1)])
    return out


def to_json(plan: dict) -> str:
    return json.dumps(plan, indent=2, sort_keys=True)


def plan_hosts(plan: dict) -> list:
    """the hosts a plan of several sources has steps for, in order of first appearance ([] for a one-source plan)"""
    return list(dict.fromkeys(check_host_name(s["host"]) for s in plan["steps"] if "host" in s))


def to_shell(plan: dict, host=None) -> str:
    """The same plan as the commands the M1 rollback script runs (m1_rollback.sh:95-99), for dry runs.  host: only that
    host's steps (a plan of several sources runs one script per host)."""
    lines = ["#!/bin/sh", "set -e"]
    if host is not None:
        check_host_name(host)
    for s in plan["steps"]:
        if host is not None and s.get("host") != host:
            continue
        if s["op"] == "rename":
            lines.append("mv -- %s %s" % (shlex.quote(s["from"]), shlex.quote(s["to"])))
        elif s["op"] == "restore_snapshot_dir":
            # the directory is only ever a single-quoted ARGUMENT of the `:` no-op (see below)
            lines.append(": restore-dir-from-pre-attack-snapshot %s" % shlex.quote(s["dir"]))
        else:
            # never a comment: a newline inside a path would end the comment and start a command.  `:` is the
            # POSIX no-op; the path is only ever a single-quoted ARGUMENT (newlines inside '...' are literal).
            lines.append(": restore-from-pre-attack-snapshot %s" % shlex.quote(s["path"]))
    return "\n".join(lines) + "\n"


def from_pipeline(g, result, attack_id=None, host_names=None) -> dict:
    """g: TemporalGraph built from a trace; result: pipeline.PipelineResult.  host_names: source id -> host name for a
    graph of several sources (g.meta["node_source"]); None: a one-source plan without host fields."""
    score = result.node_score.detach().cpu().numpy() if hasattr(result.node_score, "detach") else result.node_score
    hosts = None if host_names is None else np.asarray(host_names, object)[np.asarray(g.meta["node_source"], np.int64)]
    return undo_plan(g.meta["names"], result.plan_nodes, scores=result.plan.scores, attack_id=attack_id,
                     size_mb=g.meta.get("size_mb"), node_score=score, truncated=getattr(result.plan, "truncated", False),
                     remaining_candidates=getattr(result.plan, "remaining_candidates", 0),
                     restores=getattr(result, "restores", None), hosts=hosts,
                     evidence=getattr(result, "evidence", None), host_names=host_names,
                     sequence_evidence=getattr(result, "sequence_evidence", None),
                     incidents=getattr(result, "incidents", None), step_incident=getattr(result, "step_incident", None),
                     file_recovery=getattr(result, "file_recovery", None),
                     contamination=getattr(result, "contamination", None))
