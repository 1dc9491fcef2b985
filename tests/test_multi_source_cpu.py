"""Several sources (one tracker per node) on the host: the relabelling that defines them, the host path resolution and
interning with a source column against an event-by-event loop, the source-qualified hashes, source ids, and the
per-host plan emitter.  No GPU needed."""
import numpy as np
import pytest

from nerrf_b200 import ingest, stream, undo
from nerrf_b200._lib import NerrfError
from nerrf_b200.ai.planner import emit
from test_ingest import _tracker_style_events

pytestmark = pytest.mark.usefixtures("lib_built")


def _tracker(pid_shift=0):
    ev = _tracker_style_events()
    for e in ev:
        e["pid"] += pid_shift
    return ingest.decode_event_batch(ingest.encode_event_batch(ev))


def _hosts(k, seed=0):
    """k tracker-style traces with the same pids and paths, each on its own source, interleaved in time"""
    parts = []
    for h in range(k):
        c = stream.with_source(_tracker(), h)
        c.ts_nanos = ((c.ts_nanos.astype(np.int64) + 1000 * h) % 1_000_000_000).astype(np.int32)
        parts.append(c)
    return stream.concat_columns(parts)


# ------------------------------------------------------------------------------------------------ event-by-event loops
def _resolve_loop(cols):
    """the most recent named event of the same (source, pid), in stable time order, or None"""
    src = cols.source if cols.source is not None else np.zeros(cols.n, np.uint16)
    last, out = {}, [None] * cols.n
    for i in np.argsort(cols.timestamp, kind="stable").tolist():
        key = (int(src[i]), int(cols.pid[i]))
        if cols.text("path", i):
            last[key] = i
        out[i] = last.get(key)
    return out


def _intern_loop(cols, order, merge):
    src = cols.source if cols.source is not None else np.zeros(cols.n, np.uint16)
    pids, files, kind, names = {}, {}, [], []
    node_p, node_f, node_g = [0] * cols.n, [0] * cols.n, [-1] * cols.n

    def stem(p):
        s, d = p.rfind("/"), p.rfind(".")
        return p[:d] if merge and d > s else p

    for i in order:
        s = int(src[i])
        if (s, int(cols.pid[i])) not in pids:
            pids[(s, int(cols.pid[i]))] = len(kind); kind.append(1); names.append((s, "pid:%d" % cols.pid[i]))
        node_p[i] = pids[(s, int(cols.pid[i]))]
        p, g = cols.text("path", i), cols.text("new_path", i)
        if (s, stem(p)) not in files:
            files[(s, stem(p))] = len(kind); kind.append(0); names.append((s, p))
        node_f[i] = files[(s, stem(p))]
        if g and merge:
            files.setdefault((s, stem(g)), node_f[i])
        elif g:
            if (s, g) not in files:
                files[(s, g)] = len(kind); kind.append(0); names.append((s, g))
            node_g[i] = files[(s, g)]
    return node_p, node_f, node_g, kind, names


@pytest.mark.parametrize("k", [1, 2, 3])
def test_resolve_columns_with_source_matches_the_loop(k):
    cols = _hosts(k)
    want = _resolve_loop(cols)
    got = ingest.resolve_columns(cols)
    keep = [i for i in range(cols.n) if want[i] is not None]
    assert got.n == len(keep)
    assert got.source.tolist() == cols.source[keep].tolist()
    assert [got.text("path", j) for j in range(got.n)] == [cols.text("path", want[i]) for i in keep]


def test_pathless_write_never_resolves_to_another_hosts_file():
    a = stream.with_source(ingest.decode_event_batch(ingest.encode_event_batch(
        [{"timestamp": 10.0, "event": "openat", "path": "/app/uploads/a.dat", "pid": 7}])), 0)
    b = stream.with_source(ingest.decode_event_batch(ingest.encode_event_batch(
        [{"timestamp": 11.0, "event": "write", "path": "", "pid": 7, "size": 5}])), 1)
    r = ingest.resolve_columns(stream.concat_columns([a, b]))
    assert r.n == 1 and r.source.tolist() == [0]                  # B's write is dropped, as a single host drops it
    r = ingest.resolve_columns(stream.concat_columns([a, stream.with_source(b, 0)]))
    assert r.n == 2                                               # on one host it resolves


@pytest.mark.parametrize("merge", [True, False])
@pytest.mark.parametrize("k", [1, 2, 3, 8])
def test_host_interning_with_source_matches_the_loop_and_the_relabelled_stream(k, merge):
    cols = ingest.resolve_columns(_hosts(k))
    order = np.argsort(cols.timestamp, kind="stable")
    node_p, node_f, node_g, kind, ne, nw = ingest.intern_nodes(cols, order, merge)
    wp, wf, wg, wkind, wnames = _intern_loop(cols, order.tolist(), merge)
    assert node_p.tolist() == wp and node_f.tolist() == wf and node_g.tolist() == wg and kind.tolist() == wkind
    if k > 1:
        assert len(set(node_p.tolist())) == k * len(set(cols.pid.tolist()))     # same pids, one process per host
    rel = stream.relabel_single_source(cols)
    rp, rf, rg, rkind, rne, rnw = ingest.intern_nodes(rel, order, merge)
    assert (rp == node_p).all() and (rf == node_f).all() and (rg == node_g).all() and (rkind == kind).all()
    assert (rne == ne).all() and (rnw == nw).all()


def test_rename_aliases_only_within_its_source():
    ev_a = [{"timestamp": 1.0, "event": "openat", "path": "/d/x.dat", "pid": 5},
            {"timestamp": 2.0, "event": "rename", "path": "/d/x.dat", "new_path": "/d/y.lockbit3", "pid": 5}]
    ev_b = [{"timestamp": 3.0, "event": "openat", "path": "/d/y.txt", "pid": 5}]
    a = stream.with_source(ingest.decode_event_batch(ingest.encode_event_batch(ev_a)), 0)
    b = stream.with_source(ingest.decode_event_batch(ingest.encode_event_batch(ev_b)), 1)
    two = ingest.intern_nodes(stream.concat_columns([a, b]))
    one = ingest.intern_nodes(stream.concat_columns([a, stream.with_source(b, 0)]))
    assert two[1].tolist() == [1, 1, 3]                            # B's /d/y is a file of its own
    assert one[1].tolist() == [1, 1, 1]                            # on one host the rename target aliases it


def test_relabel_helper():
    cols = _hosts(2)
    rel = stream.relabel_single_source(cols)
    assert rel.source is None and rel.n == cols.n
    keys = set(zip(cols.source.tolist(), cols.pid.tolist()))
    assert len(set(rel.pid.tolist())) == len(keys)
    for i in range(cols.n):
        for name in ("path", "new_path"):
            t = cols.text(name, i)
            assert rel.text(name, i) == ("@%d/%s" % (cols.source[i], t) if t else "")
    assert (rel.path_flags == cols.path_flags).all()
    one = _tracker()
    assert stream.relabel_single_source(one) is one


# ------------------------------------------------------------------------------------------------------------- hashes
# today's values (the hashes before sources existed), pinned
_TODAY = {"/app/uploads/a.dat": (1552320993523368278, -7933854607864315875),
          "pid:454": (8479314093082153798, 8479314093082153798),
          "": (-1166397803181037274, -1166397803181037274),
          "/app/uploads": (-7933854607864315875, -7456019351643928870)}


def test_hashes_at_source_zero_are_todays():
    for name, (nh, dh) in _TODAY.items():
        assert stream.name_hash(name) == stream.name_hash(name, source=0) == nh
        assert stream.dir_hash(name) == stream.dir_hash(name, source=0) == dh


def test_hashes_are_qualified_by_source():
    for name in _TODAY:
        hs = {stream.name_hash(name, source=s) for s in (0, 1, 2, 65535)}
        assert len(hs) == 4
        ds = {stream.dir_hash(name, source=s) for s in (0, 1, 2, 65535)}
        assert len(ds) == 4
    # the directory hash of a file is the name hash of its directory, per source
    assert stream.dir_hash("/app/uploads/a.dat", 3) == stream.name_hash("/app/uploads", 3)


# ---------------------------------------------------------------------------------------------------------- source ids
@pytest.mark.parametrize("s", [0, 1, 65535])
def test_source_ids_in_range(s):
    cols = stream.with_source(_tracker(), s)
    assert cols.source.dtype == np.uint16 and int(cols.source[0]) == s
    stream.name_hash("/a", s)
    assert ingest.intern_nodes(cols)[3].shape[0] == ingest.intern_nodes(_tracker())[3].shape[0]


@pytest.mark.parametrize("s", [65536, -1, 1 << 20])
def test_source_ids_out_of_range_are_refused(s):
    with pytest.raises(NerrfError, match="out of range"):
        stream.with_source(_tracker(), s)
    with pytest.raises(NerrfError, match="out of range"):
        stream.name_hash("/a", s)


def test_source_registry_names():
    sp = stream.StreamingPlanner(None, None)
    assert sp.add_source("node-a") == 0 and sp.add_source("node_b.1") == 1 and sp.add_source("node-a") == 0
    assert sp.host_name(1) == "node_b.1" and sp.host_name(7) == "7"
    for bad in ("", "a;b", "a/b", "a\nb", "..", ".", "x" * 65, "a b", "$(id)", None):
        with pytest.raises(ValueError):
            sp.add_source(bad)
    assert sp.add_source("x" * 64) == 2


# ------------------------------------------------------------------------------------------------------------- emitter
def _plan(hosts=None):
    names = ["/h/a.lockbit3", "pid:3", "/h/b.dat", "/h/c.dat", "/h/d.lockbit3"]
    restores = [{"position": 1, "dir": "/h", "covers": [2, 3]}]
    return emit.undo_plan(names, [0, 4], scores=[3.0, 2.0, 1.0, 0.5], restores=restores, hosts=hosts)


def test_single_source_plan_is_unchanged():
    plan = _plan()
    assert all("host" not in s for s in plan["steps"])
    assert emit.to_json(plan) == emit.to_json(emit.undo_plan(
        ["/h/a.lockbit3", "pid:3", "/h/b.dat", "/h/c.dat", "/h/d.lockbit3"], [0, 4], scores=[3.0, 2.0, 1.0, 0.5],
        restores=[{"position": 1, "dir": "/h", "covers": [2, 3]}]))
    assert emit.plan_hosts(plan) == []
    assert emit.to_shell(plan) == ("#!/bin/sh\nset -e\nmv -- /h/a.lockbit3 /h/a.dat\n"
                                   ": restore-dir-from-pre-attack-snapshot /h\nmv -- /h/d.lockbit3 /h/d.dat\n")


def test_host_fields_and_per_host_scripts():
    plan = _plan(hosts=["nodeA", "nodeA", "nodeB", "nodeB", "nodeB"])
    assert [s["host"] for s in plan["steps"]] == ["nodeA", "nodeB", "nodeB"]
    assert emit.plan_hosts(plan) == ["nodeA", "nodeB"]
    a, b = emit.to_shell(plan, host="nodeA"), emit.to_shell(plan, host="nodeB")
    assert "a.lockbit3" in a and "d.lockbit3" not in a and "restore-dir" not in a
    assert "d.lockbit3" in b and "restore-dir" in b and "a.lockbit3" not in b


@pytest.mark.parametrize("bad", ["a;rm -rf /", "a/b", "a\nb", "..", ".", "", "x" * 65, "a'b"])
def test_hostile_host_names_are_refused(bad):
    with pytest.raises(ValueError, match="bad host name"):
        _plan(hosts=[bad] * 5)
    with pytest.raises(ValueError, match="bad host name"):
        emit.to_shell(_plan(), host=bad)
    with pytest.raises(ValueError, match="bad host name"):
        undo.parse_traces(["%s=x.pb" % bad, "ok=y.pb"])


def test_restore_covering_two_hosts_is_refused():
    names = ["/h/b.dat", "/h/c.dat"]
    with pytest.raises(ValueError, match="several hosts"):
        emit.undo_plan(names, [], restores=[{"position": 0, "dir": "/h", "covers": [0, 1]}], hosts=["a", "b"])


def test_host_graph_directory_hashes_are_per_host():
    from nerrf_b200 import pipeline
    ev = [{"timestamp": 1.0 + k, "event": "openat", "path": "/app/uploads/f%d.dat" % k, "pid": 9} for k in range(3)]
    one = ingest.decode_event_batch(ingest.encode_event_batch(ev))
    g = ingest.graph_from_columns(stream.concat_columns([stream.with_source(one, 0), stream.with_source(one, 1)]))
    files = np.nonzero(g.meta["node_kind"] == 0)[0]
    dh = pipeline.node_dir_hashes(g, files).numpy()
    src = g.meta["node_source"][files]
    assert np.unique(dh[src == 0]).size == 1 and np.unique(dh[src == 1]).size == 1 and dh[src == 0][0] != dh[src == 1][0]
    assert dh[src == 0][0] == stream.dir_hash("/app/uploads/f0.dat")                      # source 0: the plain hash
    g1 = ingest.graph_from_columns(one)                           # one source: the hashes it always had
    assert pipeline.node_dir_hashes(g1).tolist() == [stream.dir_hash(n) for n in g1.meta["names"]]


def test_cli_script_outputs_fit_the_traces():
    undo.check_outputs([("a", "a.pb"), ("b", "b.pb")], None, "dir")
    undo.check_outputs([(None, "a.pb")], "plan.sh", None)
    undo.check_outputs([("a", "a.pb")], "plan.sh", "dir")
    with pytest.raises(SystemExit, match="--shell-dir"):
        undo.check_outputs([("a", "a.pb"), ("b", "b.pb")], "plan.sh", None)     # one script would mix the hosts' commands
    with pytest.raises(SystemExit, match="HOST=PATH"):
        undo.check_outputs([(None, "a.pb")], None, "dir")


def test_second_source_after_single_source_ticks_is_refused():
    sp = stream.StreamingPlanner(None, None)
    sp.add_source("a")
    sp._host_keys = False                                         # what the first tick of a one-source feed decides
    assert sp.add_source("a") == 0
    with pytest.raises(ValueError, match="register every source"):
        sp.add_source("b")


def test_cli_trace_arguments():
    assert undo.parse_traces(["a.pb"]) == [(None, "a.pb")]
    assert undo.parse_traces(["nodeA=a.pb", "nodeB=b.pb"]) == [("nodeA", "a.pb"), ("nodeB", "b.pb")]
    with pytest.raises(SystemExit):
        undo.parse_traces(["a.pb", "nodeB=b.pb"])
    with pytest.raises(SystemExit):
        undo.parse_traces(["n=a.pb", "n=b.pb"])


def test_host_streams_collide_on_purpose():
    hs = stream.host_streams(3, 6, 2, seed=1)
    assert [int(c.source[0]) for c, _, _ in hs] == [0, 1, 2]
    (c0, enc0, att0), (c1, enc1, att1), (c2, enc2, att2) = hs
    assert att0 and not att1 and att0 == att2 and enc0 == enc2 and not enc1
    assert set(c0.pid.tolist()) & set(c1.pid.tolist()) >= {int(p[4:]) for p in att0}   # host 1's benign pids = host 0's attackers
    assert set(c0.texts("path")) & set(c1.texts("path"))
    base, _ = stream.fleet_columns(6, 2, seed=1)
    assert np.array_equal(c0.pid, base.pid) and np.array_equal(c0.strings["path"][1], base.strings["path"][1])
