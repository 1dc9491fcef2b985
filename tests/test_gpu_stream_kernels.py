"""The integer half of the live stream (needs an H100), kernel by kernel against numpy at the sizes where its tiles,
carries and 32-bit totals change over: the radix sort (csrc/radix_sort.cuh, tiles of 4096 pairs, a 256 x tiles histogram),
the exclusive scan and its max-scan twin (csrc/scan.cuh, csrc/live_stream.cu: tiles of 1024, tile sums combined 1024 at
a time with a carry, so the carry first runs above 2^20 scanned elements), nerrf_trace_stream_order (time order, pid
regroup, path resolution, retention), the device decoder with its 32-lane path-flag scan, and nerrf_trace_gather_rows.
Everything here is index work, byte copies or bit-rounded float64: every comparison is exact."""
import ctypes as C

import numpy as np
import pytest
import torch

from nerrf_b200 import _lib, ingest, stream
from nerrf_b200._lib import NerrfError
from test_gpu_graph import _check as _csr_check
from test_gpu_live_stream import _same_columns, _same_graph

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("lib_built")]

SCAN_CHUNK = 1024 * 1024             # scanned elements after which scan_sums / maxscan_sums hand a carry to the next chunk
SORT_CHUNK = 4096 * 4096             # sorted pairs after which the radix histogram (256 per tile of 4096) does
SMALL = [1, 2, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025, 4095, 4096, 4097, 16383, 16384, 16385]
BASE = 1_700_000_000


# ------------------------------------------------------------------------------------- nerrf_trace_stream_order vs numpy
def _order_dev(ts_sec, ts_nanos, pid, path_off, horizon):
    """nerrf_trace_stream_order called the way DeviceStream._rebuild calls it -> its outputs on the host"""
    n = int(ts_sec.shape[0])
    up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).cuda()
    d_sec, d_nan, d_off = up(ts_sec, np.int64), up(ts_nanos, np.int32), up(path_off, np.int64)
    d_pid = up(np.ascontiguousarray(pid, np.uint32).view(np.int32), np.int32)
    h = _lib.lib()
    need = C.c_int64()
    _lib.check(h.nerrf_trace_stream_order_workspace_bytes(n, C.byref(need)), "stream_order_workspace_bytes")
    ws = torch.empty(need.value + 256, dtype=torch.uint8, device="cuda")
    e = lambda dt: torch.empty(max(n, 1), dtype=dt, device="cuda")
    ts, order, ts_sorted, src, retain = e(torch.float64), e(torch.int64), e(torch.float64), e(torch.int64), e(torch.int64)
    res_off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    counts = (C.c_int64 * 3)()
    _lib.check(h.nerrf_trace_stream_order(n, _lib.ptr(d_sec), _lib.ptr(d_nan), _lib.ptr(d_pid), _lib.ptr(d_off), float(horizon),
                                          _lib.ptr(ts), _lib.ptr(order), _lib.ptr(ts_sorted), _lib.ptr(src), _lib.ptr(res_off),
                                          _lib.ptr(retain), counts, C.c_void_p((ws.data_ptr() + 255) & ~255), need.value,
                                          _lib.current_stream_ptr()), "nerrf_trace_stream_order")
    nk, nr = int(counts[0]), int(counts[1])
    assert 0 <= nk <= n and 0 <= nr <= n
    host = lambda t, k: t[:k].cpu().numpy()
    return {"counts": tuple(int(c) for c in counts), "ts": host(ts, n), "src": host(src, n), "order": host(order, nk),
            "ts_sorted": host(ts_sorted, nk), "res_path_off": host(res_off, n + 1), "retain": host(retain, nr)}


def _order_ref(ts_sec, ts_nanos, pid, path_off, horizon):
    """The same outputs in numpy: stable time order, stable regroup by unsigned pid, every event's path from its pid's
    latest named event at or before it in (time, stored) order, retention at the horizon."""
    n = int(ts_sec.shape[0])
    pid = np.ascontiguousarray(pid, np.uint32)
    ts = ts_sec.astype(np.float64) + ts_nanos.astype(np.float64) * 1e-9
    tord = np.argsort(ts, kind="stable")
    byp = tord[np.argsort(pid[tord], kind="stable")]
    j = np.arange(n)
    pg = pid[byp]
    start = np.r_[True, pg[1:] != pg[:-1]]
    first = np.maximum.accumulate(np.where(start, j, 0))                # regroup position of the pid's first event
    plen = path_off[1:] - path_off[:-1]
    named = plen[byp] > 0
    last_named = np.maximum.accumulate(np.where(named, j, -1))
    src = np.empty(n, np.int64)
    src[byp] = np.where(last_named >= first, byp[np.maximum(last_named, 0)], -1)
    order = tord[src[tord] >= 0]
    res_off = np.zeros(n + 1, np.int64)
    np.cumsum(np.where(src >= 0, plen[np.maximum(src, 0)], 0), out=res_off[1:])
    keep = ts > horizon
    old_named = np.maximum.accumulate(np.where(named & ~(ts[byp] > horizon), j, -1))
    end = np.r_[start[1:], True]
    pick = end & (old_named >= first)                                   # per pid: its latest named event not after the horizon
    keep[byp[old_named[pick]]] = True
    retain = np.nonzero(keep)[0]
    return {"counts": (int(order.shape[0]), int(retain.shape[0]), int(res_off[-1])), "ts": ts, "src": src, "order": order,
            "ts_sorted": ts[order], "res_path_off": res_off, "retain": retain}


def _order_loop(ts_sec, ts_nanos, pid, path_off, horizon):
    """The spec once more, event by event (small traces): pins _order_ref itself."""
    n = len(ts_sec)
    ts = [float(np.float64(int(s)) + np.float64(int(k)) * 1e-9) for s, k in zip(ts_sec, ts_nanos)]
    tord = sorted(range(n), key=lambda i: (ts[i], i))
    last, old, src = {}, {}, [-1] * n
    for i in tord:
        p = int(pid[i]) & 0xffffffff
        if path_off[i + 1] > path_off[i]:
            last[p] = i
            if not ts[i] > horizon:
                old[p] = i
        src[i] = last.get(p, -1)
    order = [i for i in tord if src[i] >= 0]
    off = [0]
    for i in range(n):
        off.append(off[-1] + (int(path_off[src[i] + 1] - path_off[src[i]]) if src[i] >= 0 else 0))
    retain = sorted({i for i in range(n) if ts[i] > horizon} | set(old.values()))
    i8 = lambda v: np.asarray(v, np.int64).reshape(-1)
    return {"counts": (len(order), len(retain), off[-1]), "ts": np.asarray(ts, np.float64).reshape(-1), "src": i8(src),
            "order": i8(order), "ts_sorted": np.asarray([ts[i] for i in order], np.float64).reshape(-1), "res_path_off": i8(off),
            "retain": i8(retain)}


def _same_order(got, want, tag=""):
    assert got["counts"] == want["counts"], (tag, got["counts"], want["counts"])
    for k in ("ts", "src", "order", "ts_sorted", "res_path_off", "retain"):
        g, w = got[k], want[k]
        if g.dtype == np.float64:
            g, w = g.view(np.uint64), w.view(np.uint64)
        assert g.shape == w.shape, (tag, k, g.shape, w.shape)
        if not np.array_equal(g, w):
            at = int(np.nonzero(g != w)[0][0])
            raise AssertionError(f"{tag}: {k}[{at}] = {got[k][at]!r}, want {want[k][at]!r} ({int((g != w).sum())} of {g.shape[0]} differ; "
                                 f"scan tile {at // 1024}, sort tile {at // 4096})")


def _check_order(sec, nanos, pid, off, horizon, tag=""):
    want = _order_ref(sec, nanos, pid, off, horizon)
    got = _order_dev(sec, nanos, pid, off, horizon)
    _same_order(got, want, tag)
    return got


def _pids(kind, n, rng):
    if kind == "one":
        return np.full(n, 0x80000007, np.uint32)
    if kind == "own":                                                   # a bijection of 2^32: every event its own pid, top bit included
        return (rng.permutation(n).astype(np.uint64) * np.uint64(2654435761) % np.uint64(1 << 32)).astype(np.uint32)
    if kind == "edge":                                                  # the sort key is the UNSIGNED pid; torch holds it as int32
        return np.array([0, 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1], np.uint32)[rng.integers(0, 5, n)]
    assert kind == "few"
    return (rng.integers(0, 8, n).astype(np.uint64) * np.uint64(0x20000001)).astype(np.uint32)


def _times(kind, n, rng):
    if kind == "equal":
        return np.full(n, BASE, np.int64), np.full(n, 5, np.int32)
    if kind == "ties":                                                  # 16 distinct timestamps, shared across pids and tiles
        return BASE + rng.integers(0, 4, n), (rng.integers(0, 4, n) * 250_000_000).astype(np.int32)
    if kind == "signed":                                                # negative seconds, nanos outside [0, 1e9)
        return rng.integers(-5, 5, n), rng.integers(-2_000_000_000, 2_000_000_000, n).astype(np.int32)
    if kind == "huge53":                                                # distinct inputs round to equal float64
        return (1 << 53) + rng.integers(-4, 5, n), rng.integers(0, 3, n).astype(np.int32)
    if kind == "huge62":
        return (1 << 62) + rng.integers(-2048, 2049, n), rng.integers(0, 1_000_000_000, n).astype(np.int32)
    sec, nanos = BASE + rng.integers(0, 60, n), rng.integers(0, 1_000_000_000, n).astype(np.int32)
    if kind in ("sorted", "reversed"):
        o = np.lexsort((nanos, sec))
        sec, nanos = sec[o], nanos[o]
        if kind == "reversed":
            sec, nanos = sec[::-1].copy(), nanos[::-1].copy()
    else:
        assert kind == "random"
    return sec, nanos


def _pid_firsts(sec, nanos, pid):
    """stored index of every pid's first event in (time, stored) order"""
    ts = sec.astype(np.float64) + nanos.astype(np.float64) * 1e-9
    tord = np.argsort(ts, kind="stable")
    byp = tord[np.argsort(pid[tord], kind="stable")]
    pg = pid[byp]
    return byp[np.r_[True, pg[1:] != pg[:-1]]]


def _path_off(kind, n, rng, sec, nanos, pid):
    if kind == "all":
        named = np.ones(n, bool)
    elif kind == "none":
        named = np.zeros(n, bool)
    elif kind == "random":
        named = rng.random(n) < 0.3
    elif kind == "first_only":                                          # one value carried down the whole pid segment
        named = np.zeros(n, bool)
        named[_pid_firsts(sec, nanos, pid)] = True
    else:
        assert kind == "first_pathless"                                 # the previous pid's path must not leak in
        named = rng.random(n) < 0.6
        named[_pid_firsts(sec, nanos, pid)] = False
    off = np.zeros(n + 1, np.int64)
    np.cumsum(np.where(named, rng.integers(1, 40, n), 0), out=off[1:])
    return off


def _trace(n, seed, pids, named, times):
    rng = np.random.default_rng(seed)
    pid = _pids(pids, n, rng)
    sec, nanos = _times(times, n, rng)
    return sec, nanos, pid, _path_off(named, n, rng, sec, nanos, pid)


def _horizons(sec, nanos, rng):
    """-inf, +inf, below all, above all, and one equal to a timestamp of the trace (`>` is strict)"""
    ts = sec.astype(np.float64) + nanos.astype(np.float64) * 1e-9
    return [-np.inf, np.inf, float(ts.min()) - 1.0, float(ts.max()) + 1.0, float(ts[rng.integers(0, ts.shape[0])])]


GRID = [(p, m, t) for p in ("one", "own", "edge", "few") for m in ("all", "none", "random", "first_only", "first_pathless")
        for t in ("random", "equal", "sorted", "reversed", "ties")] + [("few", "random", t) for t in ("signed", "huge53", "huge62")] \
    + [("edge", "first_pathless", "signed"), ("one", "first_only", "huge62")]


def test_numpy_restatement_equals_the_event_by_event_spec():
    rng = np.random.default_rng(0)
    for k, (p, m, t) in enumerate(GRID):
        for n in (1, 2, 7, 61):
            sec, nanos, pid, off = _trace(n, 1000 + k, p, m, t)
            for h in _horizons(sec, nanos, rng):
                _same_order(_order_ref(sec, nanos, pid, off, h), _order_loop(sec, nanos, pid, off, h), f"{p}/{m}/{t} n={n} h={h}")


@pytest.mark.parametrize("n", SMALL)
def test_stream_order_at_warp_tile_and_histogram_boundaries(n):
    """every pid / naming / clock shape at sizes around a warp, a scan tile (1024), a sort tile (4096) and the first
    histogram that spans two scan tiles (16384 pairs); horizon equal to a shared timestamp, and one of the others in turn"""
    rng = np.random.default_rng(n)
    for k, (p, m, t) in enumerate(GRID):
        sec, nanos, pid, off = _trace(n, 7 * n + k, p, m, t)
        hs = _horizons(sec, nanos, rng)
        for h in (hs[4], hs[k % 4]):
            got = _check_order(sec, nanos, pid, off, h, f"{p}/{m}/{t} n={n} h={h}")
            if m == "none":
                assert got["counts"][0] == 0 and got["counts"][2] == 0 and not got["res_path_off"].any()
            if m == "all":
                assert got["counts"][0] == n and np.array_equal(got["src"], np.arange(n))
            if t == "equal":                                            # nothing to order by: stored order
                assert np.array_equal(got["order"], np.nonzero(got["src"] >= 0)[0])


def test_equal_timestamps_order_by_stored_index_within_a_pid():
    """a path-less event with the timestamp of its pid's named event resolves to it only when stored after it"""
    sec = np.full(5, BASE, np.int64); nanos = np.zeros(5, np.int32)
    pid = np.array([4, 4, 9, 4, 9], np.uint32)
    off = np.array([0, 0, 11, 11, 11, 14], np.int64)                     # named: event 1 (pid 4) and event 4 (pid 9)
    got = _check_order(sec, nanos, pid, off, -np.inf)
    assert got["src"].tolist() == [-1, 1, -1, 1, 4] and got["order"].tolist() == [1, 3, 4]
    assert got["res_path_off"].tolist() == [0, 0, 11, 11, 22, 25] and got["counts"] == (3, 5, 25)


def test_horizon_equal_to_a_timestamp_is_not_after_it():
    sec = np.array([10, 10, 10, 11, 9], np.int64); nanos = np.zeros(5, np.int32)
    pid = np.array([1, 2, 1, 2, 3], np.uint32)
    off = np.arange(6, dtype=np.int64) * 3                              # every event named
    got = _check_order(sec, nanos, pid, off, 10.0)
    # ts > 10: event 3 alone; kept besides: each pid's latest named event at or before 10 (pid 1: the later stored of its tie)
    assert got["retain"].tolist() == [1, 2, 3, 4] and got["counts"] == (5, 4, 15)
    assert _check_order(sec, nanos, pid, off, np.nextafter(10.0, 0.0))["retain"].tolist() == [0, 1, 2, 3, 4]


@pytest.mark.parametrize("K", [1025, 4097, SCAN_CHUNK + 5])
def test_one_named_event_carried_across_tiles_and_chunks(K):
    """pid 5: a named event, then K path-less ones (the max-scan carries ONE value over K positions: across tiles, and for
    K > 2^20 across the chunks of the tile-maxima scan); pid 6: K path-less events that must NOT inherit it; pid 7: the
    same after a path-less start.  Stored order is shuffled."""
    rng = np.random.default_rng(K)
    pid = np.r_[np.full(K + 1, 5), np.full(K, 6), np.full(K + 2, 7)].astype(np.uint32)
    n = pid.shape[0]
    named = np.zeros(n, bool); named[0] = True; named[2 * K + 2] = True  # first event of pid 5, second event of pid 7
    sec = BASE + np.arange(n, dtype=np.int64) // 3; nanos = (np.arange(n) % 3 * 1000).astype(np.int32)
    p = rng.permutation(n)
    inv = np.empty(n, np.int64); inv[p] = np.arange(n)
    sec, nanos, pid, named = sec[p], nanos[p], pid[p], named[p]
    off = np.zeros(n + 1, np.int64); np.cumsum(np.where(named, 17, 0), out=off[1:])
    for h in (-np.inf, float(BASE + n // 6)):
        got = _check_order(sec, nanos, pid, off, h, f"K={K} h={h}")
        assert np.all(got["src"][pid == 5] == inv[0]) and np.all(got["src"][pid == 6] == -1)
        assert got["src"][inv[2 * K + 1]] == -1 and np.all(got["src"][inv[2 * K + 2:]] == inv[2 * K + 2])
        assert got["counts"][0] == 2 * K + 2 and got["counts"][2] == 17 * (2 * K + 2)


@pytest.mark.parametrize("named", ["first_only", "first_pathless", "random"])
def test_pid_segments_starting_on_tile_and_chunk_boundaries(named):
    """pid segments that begin at positions 1024 k - 1, 1024 k and 1024 k + 1 of the regroup, k up to 1024 (the second
    chunk of the tile-maxima scan starts at 1024 * 1024): a segment start must cut the scan exactly there"""
    starts = sorted({0} | {1024 * k + d for k in (1, 2, 3, 17, 1023, 1024) for d in (-1, 0, 1)})
    n = starts[-1] + 1500
    rng = np.random.default_rng(len(named))
    seg = np.searchsorted(np.asarray(starts), np.arange(n), "right") - 1
    pid = (seg.astype(np.uint64) * np.uint64(220_000_000)).astype(np.uint32)       # ascending with the segment, top bit set on the way
    sec, nanos = _times("random", n, rng)
    p = rng.permutation(n)
    pid = pid[p]
    off = _path_off(named, n, rng, sec, nanos, pid)
    ts = sec.astype(np.float64) + nanos.astype(np.float64) * 1e-9
    for h in (-np.inf, float(np.median(ts))):
        got = _check_order(sec, nanos, pid, off, h, f"{named} h={h}")
        firsts = _pid_firsts(sec, nanos, pid)
        assert firsts.shape[0] == len(starts)
        if named == "first_only":
            assert got["counts"][0] == n and np.array_equal(np.unique(got["src"]), np.sort(firsts))
        if named == "first_pathless":
            assert np.all(got["src"][firsts] == -1)


@pytest.mark.parametrize("n", [SCAN_CHUNK, SCAN_CHUNK + 1])
@pytest.mark.parametrize("pids,named,times", [("one", "first_only", "random"), ("one", "none", "ties"), ("few", "random", "ties"),
                                              ("own", "all", "random"), ("edge", "first_pathless", "sorted"),
                                              ("few", "random", "reversed")])
def test_stream_order_where_the_scans_enter_their_second_chunk(n, pids, named, times):
    """1024 * 1024 scanned elements fill the first chunk of scan_sums / maxscan_sums exactly; one more starts the second,
    which only has the carry to go by.  Equal-timestamp runs straddle position 2^20 (and every sort tile) in "ties"."""
    sec, nanos, pid, off = _trace(n, n % 1000, pids, named, times)
    ts = sec.astype(np.float64) + nanos.astype(np.float64) * 1e-9
    for h in (float(np.sort(ts)[n // 2]), -np.inf):
        got = _check_order(sec, nanos, pid, off, h, f"{pids}/{named}/{times} n={n} h={h}")
        if named == "none":
            assert got["counts"][0] == 0 and got["counts"][2] == 0


def test_stream_order_where_the_radix_histogram_enters_its_second_chunk():
    """16,777,216 + 8,193 events: 4,099 sort tiles, so each of the 12 passes (8 over the 64-bit time keys, 4 over the pid)
    scans a histogram of 256 * 4099 > 2^20 cells and the scan of its tile sums needs the carry.  60,000 distinct timestamps
    and 4,096 pids: long equal-key runs across sort tiles and across the chunk boundary, where only stability orders them.
    Costs about 2 GB of device memory and 3 GB of host memory, and 14 s beside an H100 80GB HBM3 (700 W limit), nearly all
    of it the numpy reference (deselect by name)."""
    n = SORT_CHUNK + 2 * 4096 + 1
    rng = np.random.default_rng(24)
    sec = BASE + rng.integers(0, 60, n); nanos = (rng.integers(0, 1000, n) * 1_000_000).astype(np.int32)
    pid = (rng.integers(0, 4096, n).astype(np.uint64) * np.uint64(1048583) % np.uint64(1 << 32)).astype(np.uint32)
    off = np.zeros(n + 1, np.int64)
    np.cumsum(np.where(rng.random(n) < 0.3, rng.integers(1, 40, n), 0), out=off[1:])
    _check_order(sec, nanos, pid, off, float(np.float64(BASE + 30) + np.float64(500_000_000) * 1e-9), "17M")


# ------------------------------------------------------------------------------------------ resolved bytes vs 2^31
def _one_pid(path_lengths):
    n = len(path_lengths)
    off = np.zeros(n + 1, np.int64); np.cumsum(np.asarray(path_lengths, np.int64), out=off[1:])
    return BASE + np.arange(n, dtype=np.int64), np.zeros(n, np.int32), np.full(n, 3, np.uint32), off


@pytest.mark.parametrize("case", ["repeated", "three_of_2^30", "one_of_2^31"])
def test_resolved_paths_of_2_31_bytes_are_refused_not_wrapped(case):
    """The resolved path column repeats a path for every path-less event after it: 4 KiB of stored path bytes resolve to
    2^31 + 4096.  Its offsets are scanned in int32, so the library must refuse -- never hand back wrapped offsets.  Only
    offsets are passed in (no string bytes exist), and only nerrf_trace_stream_order runs: it writes n + 1 offsets."""
    lengths = {"repeated": [4096] + [0] * (1 << 19), "three_of_2^30": [1 << 30] * 3, "one_of_2^31": [1 << 31]}[case]
    sec, nanos, pid, off = _one_pid(lengths)
    want = _order_ref(sec, nanos, pid, off, -np.inf)["counts"][2]
    assert want >= 1 << 31
    with pytest.raises(NerrfError, match=r"2\^31 - 1"):
        got = _order_dev(sec, nanos, pid, off, -np.inf)
        pytest.fail(f"resolved bytes {want} came back as counts[2] = {got['counts'][2]}, res_path_off[-1] = {got['res_path_off'][-1]}")
    _check_order(*_one_pid([4096, 0, 0]), -np.inf)                       # the library is usable afterwards


def test_resolved_paths_of_2_31_minus_1_bytes_are_exact():
    sec, nanos, pid, off = _one_pid([4096] + [0] * ((1 << 19) - 2) + [4095])    # (2^19 - 1) * 4096 + 4095
    got = _check_order(sec, nanos, pid, off, -np.inf)
    assert got["counts"][2] == got["res_path_off"][-1] == (1 << 31) - 1


def test_compaction_refuses_2_31_string_bytes():
    """nerrf_trace_gather_rows scans the lengths of all four string columns together in int32; compact() checks the sum
    first.  (The check is host code over four totals: the gather itself reads the bytes it sums, so reaching the limit
    through it would take 2 GiB of strings.)"""
    stream._require_gather_fits([0, 0, 0, 0])
    stream._require_gather_fits([(1 << 31) - 1, 0, 0, 0])
    stream._require_gather_fits([1 << 29, 1 << 29, 1 << 29, (1 << 29) - 1])
    for bad in ([1 << 31, 0, 0, 0], [1 << 29, 1 << 29, 1 << 29, 1 << 29], [0, 0, 1 << 40, 0]):
        with pytest.raises(NerrfError, match=r"2\^31 - 1"):
            stream._require_gather_fits(bad)
    dc, m, cols = _decoded(_wire(np.random.default_rng(5), 300))
    rows = np.random.default_rng(6).permutation(m)[:120]
    want = [int((cols.strings[k][0][rows + 1] - cols.strings[k][0][rows]).sum()) for k in ingest.STRING_COLUMNS]
    assert stream._rows_string_bytes(dc, torch.from_numpy(np.sort(rows)).cuda()) == want
    assert stream._rows_string_bytes(dc, torch.zeros(0, dtype=torch.int64, device="cuda")) == [0, 0, 0, 0]


# ------------------------------------------------------------------------ the radix sort's other client: the CSR constructor
def _edges(E, N, shape, seed):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, N, E)
    if shape == "ties":                                                  # few destinations, 8 distinct times: stability decides
        return src, rng.integers(0, min(N, 3), E), rng.integers(0, 8, E).astype(np.float32) * np.float32(7.5), np.ones(E, np.float32)
    assert shape == "time_ordered"                                      # the 3-pass path that starts at bit 32
    return src, rng.integers(0, N, E), np.sort(rng.uniform(0, 60, E).astype(np.float32)), rng.uniform(0.5, 1.0, E).astype(np.float32)


@pytest.mark.parametrize("E", [16383, 16384, 16385])
@pytest.mark.parametrize("N,shape", [(3, "ties"), ((1 << 20) + 1, "ties"), ((1 << 20) + 1, "time_ordered"), (3, "time_ordered")])
def test_csr_sort_where_the_histogram_crosses_a_scan_tile(E, N, shape):
    """N = 3 and 2^20 + 1: 34 and 53 key bits, neither a multiple of the 8 bits a pass sorts"""
    _csr_check(*_edges(E, N, shape, E + N), N)


@pytest.mark.parametrize("N,shape", [(3, "ties"), ((1 << 20) + 1, "time_ordered")])
def test_csr_sort_where_the_histogram_enters_its_second_chunk(N, shape):
    """16,777,216 + 8,193 edges = 4,099 sort tiles: the scan of the 256 * 4099 histogram cells needs its carry.  About 1 GB of
    device memory and 5 to 8 s each beside an H100 80GB HBM3 (700 W limit), most of it np.lexsort (deselect by name)."""
    E = SORT_CHUNK + 2 * 4096 + 1
    rp, _, _ = _csr_check(*_edges(E, N, shape, N), N)
    assert rp[-1] == E


# ------------------------------------------------------------------------------------------ decoder and warp_path_flags
def _varint(v):
    out = bytearray()
    while True:
        b = v & 0x7f
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def _field(num, s):
    return _varint(num << 3 | 2) + _varint(len(s)) + s


def _record(body):
    return b"\x0a" + _varint(len(body)) + body


def _text(rng, n):
    return bytes(rng.integers(97, 123, n, dtype=np.uint8))


def _wire(rng, m):
    """m tracker-like records: path-less writes, renames with a target, pids over the whole uint32 range"""
    ev = []
    for _ in range(m):
        sc = ["openat", "write", "rename", "unlink", "", "file_encrypt_start", "file_created"][int(rng.integers(7))]
        e = {"ts": (BASE + int(rng.integers(0, 90)), int(rng.integers(0, 1_000_000_000))), "pid": int(rng.integers(0, 1 << 32)),
             "tid": int(rng.integers(0, 1 << 16)), "comm": _text(rng, int(rng.integers(0, 16))), "syscall": sc,
             "path": b"" if sc == "write" else b"/app/uploads/" + _text(rng, int(rng.integers(1, 30))),
             "flags": int(rng.integers(0, 4)), "ret_val": int(rng.integers(-3, 3)), "bytes": int(rng.integers(0, 1 << 40))}
        if sc == "rename":
            e["new_path"] = e["path"] + b".lockbit3"
        ev.append(e)
    return ingest.encode_event_batch(ev)


LENGTHS = [0, 1, 31, 32, 33, 127, 128, 4096, 70000]                     # 128: the length varint grows to two bytes


def _wire_of_lengths(rng):
    """every LENGTHS value in each of the four string fields alone, and in all four at once"""
    names = ("comm", "syscall", "path", "new_path")
    ev = []
    for n in LENGTHS:
        for who in [(k,) for k in names] + [names]:
            e = {"ts": (BASE, n), "pid": 1 + n}
            for k in who:
                e[k] = _text(rng, n)
            ev.append(e)
    return ingest.encode_event_batch(ev)


def _decoded(wire):
    """-> (the device columns, rows, the host decoder's columns)"""
    raw = np.frombuffer(wire, np.uint8)
    dc = stream._DeviceColumns(torch.device("cuda"), 1, [1, 1, 1, 1])
    m, _, _ = stream._decode_into(dc, 0, [0, 0, 0, 0], raw, False)
    return dc, m, ingest.decode_event_batch(wire)


@pytest.mark.parametrize("m", [255, 256, 257])
def test_device_decoder_around_a_scan_tile_of_string_lengths(m):
    wire = _wire(np.random.default_rng(m), m)                            # 4 m scanned lengths: 1020, 1024, 1028
    _same_columns(stream.decode_event_batch_device(wire), ingest.decode_event_batch(wire))


def test_device_decoder_of_more_than_2_18_records_in_one_call():
    """4 * 263,168 scanned string lengths: the scan of their tile sums enters its second chunk"""
    wire = _wire(np.random.default_rng(18), 1024) * 257
    want = ingest.decode_event_batch(wire)
    assert 4 * want.n > SCAN_CHUNK
    _same_columns(stream.decode_event_batch_device(wire), want)


def test_device_decoder_string_lengths_up_to_70000_bytes():
    wire = _wire_of_lengths(np.random.default_rng(70))
    want = ingest.decode_event_batch(wire)
    assert sorted(set((want.strings["path"][0][1:] - want.strings["path"][0][:-1]).tolist())) == LENGTHS
    _same_columns(stream.decode_event_batch_device(wire), want)


def test_device_decoder_repeated_string_field_last_one_wins():
    rng = np.random.default_rng(2)
    recs, second = [], []
    for num in (4, 5, 6, 7):
        for n1, n2 in ((70000, 3), (200, 0), (33, 32), (5, 40)):
            a, b = _text(rng, n1), _text(rng, n2)
            recs.append(_record(b"\x10\x07" + _field(num, a) + _field(num, b)))
            second.append((num, b))
    wire = b"".join(recs)
    want = ingest.decode_event_batch(wire)
    for i, (num, b) in enumerate(second):
        off, data = want.strings[ingest.STRING_COLUMNS[num - 4]]
        assert bytes(data[off[i]:off[i + 1]]) == b
    _same_columns(stream.decode_event_batch_device(wire), want)


def _path_flags_py(s):
    low = s.lower()                                                     # bytes.lower() folds ASCII only, like the C rule
    return ((1 if b".lockbit" in s else 0) | (2 if b"readme" in low or b"ransom" in low else 0)
            | (4 if s.startswith(b"/tmp") or s.startswith(b"/proc") else 0) | (8 if s.endswith(b".lockbit3") else 0))


def test_path_flags_with_the_needle_at_every_position():
    """each needle at every start of strings of 4..12, 31..41 and 63..73 bytes -- up to the last legal start (where the
    32-lane scan's bounds `i + 6 <= n` and `i + 8 <= n` part, and across the lane 31 / lane 32 seam) and one past it, cut
    off by the end of the string, where it must not match -- with near-misses, over three fillers"""
    needles = [b".lockbit", b".lockbit3", b"README", b"readme", b"RaNsOm", b"RANSOM", b"/tmp", b"/proc",
               b".lockbi", b"READM", b"/tm", b"x.lockbit3x", b".LOCKBIT", b"/proC"]
    paths = []
    for n in list(range(4, 13)) + list(range(31, 42)) + list(range(63, 74)):
        for fill in (b"x", b"/", b"."):
            for nd in needles:
                for p in range(0, max(n - len(nd) + 2, 1)):
                    paths.append((fill * p + nd + fill * n)[:n])
    assert {_path_flags_py(s) for s in paths} >= {0, 1, 2, 4, 8 | 1}
    wire = ingest.encode_event_batch([{"ts": (BASE, 0), "pid": 1, "syscall": "openat", "path": s} for s in paths])
    want = ingest.decode_event_batch(wire)
    assert want.n == len(paths)
    spec = np.asarray([_path_flags_py(s) for s in paths], np.uint8)
    assert np.array_equal(ingest.path_flags_of(*want.strings["path"]), spec) and np.array_equal(want.path_flags, spec)
    got = stream.decode_event_batch_device(wire)
    bad = np.nonzero(got.path_flags != spec)[0]
    assert bad.size == 0, [(paths[i], int(got.path_flags[i]), int(spec[i])) for i in bad[:5]]
    _same_columns(got, want)


# ------------------------------------------------------------------------------------------------ nerrf_trace_gather_rows
def _gather_dev(dc, rows):
    m = int(rows.shape[0])
    out = stream._DeviceColumns(dc.dev, dc.rows, [d.numel() for d in dc.data])
    d_rows = torch.from_numpy(np.ascontiguousarray(rows, np.int64)).cuda()
    need = C.c_int64()
    _lib.check(_lib.lib().nerrf_trace_gather_rows_workspace_bytes(m, C.byref(need)), "gather_rows_workspace_bytes")
    ws = torch.empty(need.value + 256, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib().nerrf_trace_gather_rows(dc.ptrs(), _lib.ptr(d_rows) if m else None, m, out.ptrs(),
                                                  C.c_void_p((ws.data_ptr() + 255) & ~255), need.value, _lib.current_stream_ptr()),
               "nerrf_trace_gather_rows")
    return out.host(m)


def _gather_ref(cols, rows):
    sc = {k: getattr(cols, k)[rows] for k in ("ts_sec", "ts_nanos", "pid", "tid", "flags", "ret_val", "bytes", "event_slot", "path_flags")}
    strings = {k: ingest._gather_strings(*cols.strings[k], rows) for k in ingest.STRING_COLUMNS}
    return ingest.EventColumns(n=int(rows.shape[0]), strings=strings, **sc)


def _row_sets(m, rng):
    some = np.sort(rng.permutation(m)[:max(m // 3, 1)])
    return {"none": np.zeros(0, np.int64), "all": np.arange(m), "first": np.array([0]), "last": np.array([m - 1]),
            "every_other": np.arange(0, m, 2), "odd": np.arange(1, m, 2), "random": some, "reversed": np.arange(m)[::-1].copy()}


@pytest.mark.parametrize("m", [255, 256, 257])
def test_gather_rows_around_a_scan_tile_with_empty_and_long_strings(m):
    rng = np.random.default_rng(m)
    long = _wire_of_lengths(rng)                                         # 45 records: strings of 0 .. 70,000 bytes
    dc, rows, cols = _decoded(_wire(rng, m - 45 - 20) + long + _wire(rng, 20))
    assert rows == m
    for name, idx in _row_sets(m, rng).items():
        _same_columns(_gather_dev(dc, idx), _gather_ref(cols, idx))


def test_gather_rows_of_more_than_2_18_rows():
    rng = np.random.default_rng(19)
    dc, m, cols = _decoded(_wire(rng, 1024) * 257 + _wire_of_lengths(rng))
    assert 4 * m > SCAN_CHUNK
    for name, idx in _row_sets(m, rng).items():
        _same_columns(_gather_dev(dc, idx), _gather_ref(cols, idx))


def test_append_compact_append_with_more_than_2_20_resident_events():
    """the live stream where its scans and sorts run past 2^20 elements: a 12,000-process fleet trace (1.25 M events) in
    two appends with a compaction that keeps more than 2^20 rows between them, against the whole-trace DeviceStream"""
    cols, _ = stream.fleet_columns(12000, 40, seed=5)
    recs = ingest.encode_columns(cols)
    order = np.argsort(cols.timestamp, kind="stable")
    cut = int(0.93 * cols.n)
    first, second = b"".join(recs[i] for i in order[:cut]), b"".join(recs[i] for i in order[cut:])
    ref = stream.DeviceStream(ingest.decode_event_batch(first + second), "cuda", observable=True)
    t0, t1 = ref.span()
    ds = stream.DeviceStream.live("cuda", observable=True)
    ds.append(first)
    assert ds.resident_events == cut
    ds.compact(t0 + 1.0)
    assert SCAN_CHUNK < ds.resident_events < cut
    ds.append(second)
    assert ds.resident_events > SCAN_CHUNK and ds.span()[1] == t1
    for lo, hi in [(t0 + 1.0, t0 + 2.5), (t0 + 50.0, t0 + 50.5), (t1 - 1.0, t1)]:
        _same_graph(ds.window_graph(lo, hi, 60.0), ref.window_graph(lo, hi, 60.0))
    g, w = ds.window_graph(t0 + 1.0, t1, 60.0), ref.window_graph(t0 + 1.0, t1, 60.0)      # every resident event, names aside
    assert g.meta["events"] == w.meta["events"] > SCAN_CHUNK and g.num_nodes == w.num_nodes
    assert torch.equal(g.rowptr, w.rowptr) and torch.equal(g.col, w.col)
    assert torch.equal(g.ew.view(torch.int32), w.ew.view(torch.int32)) and torch.equal(g.x.view(torch.int32), w.x.view(torch.int32))
    assert torch.equal(g.meta["name_hash"], w.meta["name_hash"]) and np.array_equal(g.meta["label"], w.meta["label"])
