"""Restore candidates on the host: the undo-plan emitter's directory-restore step, the parent-directory hash and the
restore proposal (collateral) of the pipeline.  CPU only."""
import json
import subprocess

import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G, pipeline, stream, trace_sim
from nerrf_b200.ai.planner import emit


def _fnv_mix(b: bytes) -> int:
    """Independent statement of the name hash: FNV-1a seeded with the length, murmur3 finaliser, never 0, signed."""
    m = (1 << 64) - 1
    h = 0xcbf29ce484222325 ^ len(b)
    for c in b:
        h = ((h ^ c) * 0x100000001b3) & m
    for mul in (0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53):
        h ^= h >> 33
        h = (h * mul) & m
    h ^= h >> 33
    h = h or 1
    return h - (1 << 64) if h >= (1 << 63) else h


@pytest.mark.parametrize("name,parent", [("/app/uploads/a_001.dat", "/app/uploads"), ("/a", ""), ("noslash", ""),
                                         ("/x/y/", "/x/y"), ("/d/é ü.lockbit3", "/d"), ("//", "/")])
def test_dir_hash_is_the_name_hash_of_the_parent(name, parent):
    assert stream.parent_dir(name) == parent
    assert stream.dir_hash(name) == stream.name_hash(parent) == _fnv_mix(parent.encode())
    assert stream.dir_hash("pid:454") == stream.name_hash("pid:454")


def test_encrypted_twin_shares_the_directory():
    assert stream.dir_hash("/app/uploads/x.dat") == stream.dir_hash("/app/uploads/x.lockbit3") != stream.dir_hash("/app/x.dat")


def _two_dir_graph():
    events = trace_sim.lockbit_trace(n_files=6, seed=3, benign_files=3)
    for i, e in enumerate(trace_sim.lockbit_trace(n_files=0, seed=4, benign_files=2, pid=900)):
        if e["event"] == "file_created":
            e = dict(e, path=e["path"].replace("/app/uploads/", "/srv/data/"), size=(i + 1) << 20)
            events.append(e)
    events.sort(key=lambda e: e["timestamp"])
    return G.graph_from_events(events)


def test_collateral_is_the_size_of_the_directory_files_that_are_not_candidates():
    g = _two_dir_graph()
    names, kind, size = g.meta["names"], np.asarray(g.meta["node_kind"]), np.asarray(g.meta["size_mb"], np.float32)
    files = np.nonzero(kind == 0)[0]
    up = [int(n) for n in files if names[n].startswith("/app/uploads/") and "." in names[n].rsplit("/", 1)[1]
          and "README" not in names[n]]
    srv = [int(n) for n in files if names[n].startswith("/srv/data/")]
    assert len(up) == 9 and len(srv) == 2
    cand = np.array(up[:7] + srv[:1], np.int64)                           # 7 of 9 upload files, 1 of 2 /srv files
    dirs, coll, slot = pipeline.propose_restores(pipeline.node_dir_hashes(g, cand), pipeline.node_dir_hashes(g, files),
                                                 size[files], torch.from_numpy(np.isin(files, cand)), max_restores=4,
                                                 min_files=2)
    assert dirs.tolist() == [stream.dir_hash("/app/uploads/x")]           # /srv/data has one candidate: below min_files
    others = [int(n) for n in files if stream.parent_dir(names[n]) == "/app/uploads" and int(n) not in cand]
    assert set(up[7:]) <= set(others)
    assert coll[0] == np.float32(np.float64(size[others]).sum())
    assert slot.tolist() == [0] * 7 + [-1]
    # ranking: most candidates first, at most max_restores
    dirs2, _, slot2 = pipeline.propose_restores(pipeline.node_dir_hashes(g, cand), pipeline.node_dir_hashes(g, files),
                                                size[files], torch.from_numpy(np.isin(files, cand)), max_restores=1, min_files=1)
    assert dirs2.tolist() == dirs.tolist() and slot2.tolist() == slot.tolist()
    none = pipeline.propose_restores(pipeline.node_dir_hashes(g, cand), pipeline.node_dir_hashes(g, files), size[files],
                                     torch.from_numpy(np.isin(files, cand)), min_files=8)
    assert none[0].size == 0 and (none[2] == -1).all()


def test_restore_step_in_json_and_shell(tmp_path):
    names = {0: "/app/uploads/a.lockbit3", 1: "pid:454", 2: "/app/uploads/b.lockbit3", 3: "/tmp/x.txt"}
    restores = [{"position": 0, "dir": "/app/uploads", "dir_hash": 7, "covers": [0, 2]}]
    plan = emit.undo_plan(names, [1, 3], scores=[-10.0, -5.0, -4.0, -3.5], restores=restores)
    kinds = [s["op"] for s in plan["steps"]]
    assert kinds == ["restore_snapshot_dir", "restore_snapshot", "restore_snapshot"]
    st = plan["steps"][0]
    assert st["dir"] == "/app/uploads" and st["covers"] == ["/app/uploads/a.lockbit3", "/app/uploads/b.lockbit3"]
    assert [v["path"] for v in st["validate"]] == st["covers"] and all(v["check"] == "md5" for v in st["validate"])
    assert [s["order"] for s in plan["steps"]] == [0, 1, 2] and st["reward_after"] == -5.0
    assert plan["steps"][2]["reward_after"] == -3.5 and plan["reward_after"] == -3.5
    assert json.loads(emit.to_json(plan)) == plan
    script = emit.to_shell(plan)
    assert script.splitlines()[2] == ": restore-dir-from-pre-attack-snapshot /app/uploads"
    subprocess.run(["sh", "-c", script], cwd=tmp_path, check=True)


def test_plans_without_restores_are_unchanged():
    names = ["/f0.lockbit3", "/f1"]
    a = emit.undo_plan(names, np.asarray([1, 0]), scores=[-3.0, -2.0])
    assert emit.to_json(emit.undo_plan(names, np.asarray([1, 0]), scores=[-3.0, -2.0], restores=[])) == emit.to_json(a)
    assert emit.to_json(emit.undo_plan(names, np.asarray([1, 0]), scores=[-3.0, -2.0], restores=None)) == emit.to_json(a)
    assert a["version"] == emit.PLAN_VERSION == 1


def test_hostile_directory_names_cannot_inject_commands(tmp_path):
    marker = tmp_path / "PWNED"
    dirs = [f"/data/a\ntouch {marker} #", f"/data/b'; touch {marker}; '", f"/data/$(touch {marker})", f"/data/`touch {marker}`"]
    names = {i: d + "/f.lockbit3" for i, d in enumerate(dirs)}
    restores = [{"position": i, "dir": d, "covers": [i]} for i, d in enumerate(dirs)]
    plan = emit.undo_plan(names, [], restores=restores)
    assert plan["steps"][0]["hostile_name"] and "hostile_name" not in plan["steps"][2]
    script = emit.to_shell(plan)
    assert not any(l.lstrip().startswith("#") for l in script.splitlines()[1:])
    subprocess.run(["sh", "-c", script], cwd=tmp_path, check=True)
    assert not marker.exists()
    assert json.loads(emit.to_json(plan))["steps"][0]["dir"] == dirs[0]


def test_multi_gpu_refuses_restore_candidates():
    ctx = pipeline.DistContext(rank=0, world=2)
    with pytest.raises(NotImplementedError, match="one GPU"):
        pipeline.run(None, None, None, None, None, None, dist_ctx=ctx, restore_candidates=True)
    sp = stream.StreamingPlanner(None, None, dist_ctx=ctx, restore_candidates=True)
    with pytest.raises(NotImplementedError, match="one GPU"):
        sp.run(None)
