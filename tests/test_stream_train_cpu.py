"""CPU side of training on stream windows: fleet traces with bystander processes (stream.fleet_columns) and the command
line of `python -m nerrf_b200.ai.train --fleet / --stream`.  The windows themselves are built on the GPU
(tests/test_gpu_stream_train.py)."""
import hashlib

import numpy as np
import pytest

from nerrf_b200 import graph as G, ingest, stream
from nerrf_b200.ai import train as T

pytestmark = pytest.mark.usefixtures("lib_built")


def _digest(cols):
    h = hashlib.sha256()
    for k in ("ts_sec", "ts_nanos", "pid", "tid", "flags", "ret_val", "bytes", "event_slot", "path_flags"):
        a = getattr(cols, k)
        h.update(k.encode()); h.update(str(a.dtype).encode()); h.update(np.ascontiguousarray(a).tobytes())
    for k in ingest.STRING_COLUMNS:
        off, data = cols.strings[k]
        h.update(k.encode()); h.update(off.tobytes()); h.update(data.tobytes())
    return h.hexdigest()


# digests of fleet_columns as it was before it took `bystanders`: the default must keep emitting exactly these events
@pytest.mark.parametrize("procs,attacked,seed,n,digest", [
    (60, 4, 3, 6612, "2f1563124d2278231b305ad9dde3c230248c36707db04703f711e32223fe1808"),
    (25, 25, 7, 4925, "b2343e7848ac74bd4c93f16e8fe17b479b30dbc0846733af1db96237693a70ad"),
    (30, 0, 1, 3120, "b2e15ab6a841cae17fc35797c6c9d11ffeb8cf916f209355a8e2cc8fc0ecdef3")])
def test_fleet_without_bystanders_is_unchanged(procs, attacked, seed, n, digest):
    for cols in (stream.fleet_columns(procs, attacked, seed=seed)[0], stream.fleet_columns(procs, attacked, seed=seed, bystanders=0)[0]):
        assert cols.n == n and _digest(cols) == digest
    cols, _, pids = stream.fleet_columns(procs, attacked, seed=seed, return_pids=True)
    attack = np.isin(cols.event_slot, (1, 2, 3))
    assert pids == {"pid:%d" % p for p in np.unique(cols.pid[attack]).tolist()}


@pytest.mark.parametrize("k", [1, 3])
def test_fleet_bystanders_touch_encrypted_files_after_the_attacker(k):
    base, enc0, pids0 = stream.fleet_columns(40, 5, seed=2, return_pids=True)
    cols, enc, pids = stream.fleet_columns(40, 5, seed=2, return_pids=True, bystanders=k)
    assert enc == enc0 and pids == pids0                        # the same attack; only the attackers are ransomware
    new = np.setdiff1d(np.unique(cols.pid), np.unique(base.pid))
    assert new.size == 5 * k                                    # k processes of their own per attacked process
    assert not np.isin(new, base.pid).any()
    by = np.isin(cols.pid, new)
    assert set(cols.event_slot[by].tolist()) <= {4, 5}          # bystanders only open and write
    path = np.asarray(cols.texts("path"), dtype=object)
    ts = cols.timestamp
    after = 0
    for p_ in new.tolist():
        mine = np.nonzero(cols.pid == p_)[0]
        lock = [i for i in mine.tolist() if path[i] in enc]
        assert lock                                             # every bystander writes some encrypted file ...
        for i in lock:                                          # ... after its encryption completed
            done = np.nonzero((path == path[i]) & (cols.event_slot == 2))[0]
            assert done.size == 1 and ts[i] > ts[done[0]]
            after += 1
    assert after > 0
    # the host loader's edge labels now differ from "touches an encrypted file"
    w = stream.window(cols, -np.inf, np.inf)
    g = G.graph_from_events(ingest.events_from_columns(w))
    src = g.col.astype(np.int64)
    dst = np.repeat(np.arange(g.num_nodes), np.diff(g.rowptr.astype(np.int64)))
    touches_enc = (g.meta["label"][src] > 0) | (g.meta["label"][dst] > 0)
    assert (touches_enc & (g.meta["edge_label"] == 0)).any()


def test_cli_parses_the_stream_training_flags():
    a = T.parser().parse_args(["--device", "cuda", "--fleet", "400,8", "--bystanders", "2", "--windows", "16", "--edge-loss", "1.0",
                               "--out", "w.pt"])
    assert (a.fleet, a.bystanders, a.windows, a.edge_loss, a.out, a.device) == ((400, 8), 2, 16, 1.0, "w.pt", "cuda")
    assert a.stream is None and a.window_s == 60.0 and a.files_per_window == 512 and a.seed == 0
    a = T.parser().parse_args(["--device", "cuda", "--stream", "trace.pb", "--window-s", "30", "--files-per-window", "64"])
    assert (a.stream, a.fleet, a.window_s, a.files_per_window) == ("trace.pb", None, 30.0, 64)
    d = T.parser().parse_args([])                               # the toy-set path and its defaults
    assert (d.fleet, d.stream, d.traces, d.epochs, d.device, d.edge_loss) == (None, None, 8, 150, "cpu", 0.0)


@pytest.mark.parametrize("argv", [["--fleet", "8"], ["--fleet", "4,8"], ["--fleet", "a,b"],
                                  ["--fleet", "8,2", "--stream", "t.pb"]])
def test_cli_refuses_bad_stream_flags(argv, capsys):
    with pytest.raises(SystemExit):
        T.parser().parse_args(argv)


def test_cli_stream_training_needs_a_gpu_device(capsys):
    with pytest.raises(SystemExit):
        T.main(["--fleet", "8,2", "--device", "cpu"])
    assert "--device cuda" in capsys.readouterr().err
