"""Live-stream ingest on the device: the cfg-5 fleet trace (fleet_columns(10400, 40, seed=5)) encoded to EventBatch records
and fed to DeviceStream.live in batches of 1 s of trace time, with retention after every 30-s tick (60-s window).

Per append (CUDA events): framing (host), device decode, rebuild (time order + resolution + columns) and compaction;
median / p99; the device decoder's rate in GB/s of wire bytes against ingest.decode_event_batch + DeviceStream(cols)
over the same bytes; the peak resident event count; the GPU and its power limit.

    python scripts/live_stream_timing.py [n_procs] [--out file.json]
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from nerrf_b200 import ingest, stream  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def pct(v, q):
    return float(np.percentile(np.asarray(v, np.float64), q)) if len(v) else 0.0


def main():
    argv = sys.argv[1:]
    out_path = None
    if "--out" in argv:
        k = argv.index("--out")
        out_path = argv[k + 1]
        argv = argv[:k] + argv[k + 2:]
    n_procs = int(argv[0]) if argv else 10400
    info = gpu_info()
    cols, _ = stream.fleet_columns(n_procs, 40 * n_procs // 10400 or 1, seed=5)
    recs = ingest.encode_columns(cols)
    ts = cols.timestamp
    order = np.argsort(ts, kind="stable")
    key = np.floor(ts[order] - ts.min()).astype(np.int64)
    batches = [b"".join(recs[i] for i in part) for part in np.split(order, np.nonzero(np.diff(key))[0] + 1)]
    wire = b"".join(batches)

    # whole-trace reference over the same bytes: host decoder + DeviceStream(cols) (resolution, sort, upload)
    torch.cuda.synchronize()
    a = time.perf_counter(); whole = ingest.decode_event_batch(wire); t_host_dec = time.perf_counter() - a
    a = time.perf_counter(); ref = stream.DeviceStream(whole, "cuda"); torch.cuda.synchronize(); t_ds = time.perf_counter() - a
    del ref

    window, tick = 60.0, 30.0
    for rep in range(2):                                         # first pass warms the allocator and the kernels
        ds = stream.DeviceStream.live("cuda")
        frame, dec, reb, comp, peak = [], [], [], [], 0
        t_hi = None
        wall = time.perf_counter()
        for b in batches:
            ds.append(b)
            tm = ds.timings_ms
            frame.append(tm.get("frame_ms", 0.0)); dec.append(tm.get("decode_ms", 0.0)); reb.append(tm.get("rebuild_ms", 0.0))
            peak = max(peak, ds.resident_events)
            first, last = ds.span()
            t_hi = first if t_hi is None else t_hi
            while last > t_hi + tick:
                t_hi += tick
                ds.compact(t_hi - window)
                comp.append(ds.timings_ms["compact_ms"])
        torch.cuda.synchronize()
        wall = time.perf_counter() - wall
    dec_s = sum(dec) / 1e3
    res = {
        "gpu": info, "events": int(cols.n), "wire_bytes": len(wire), "appends": len(batches), "ticks": len(comp),
        "frame_ms": {"median": pct(frame, 50), "p99": pct(frame, 99)},
        "decode_ms": {"median": pct(dec, 50), "p99": pct(dec, 99)},
        "rebuild_ms": {"median": pct(reb, 50), "p99": pct(reb, 99)},
        "compact_ms": {"median": pct(comp, 50), "p99": pct(comp, 99)},
        "device_decode_GBps": len(wire) / dec_s / 1e9 if dec_s else None,
        "host_decode_GBps": len(wire) / t_host_dec / 1e9,
        "host_decode_plus_devicestream_GBps": len(wire) / (t_host_dec + t_ds) / 1e9,
        "live_wall_s": wall, "peak_resident_events": int(peak),
    }
    line = json.dumps(res)
    print(line)
    if out_path:
        with open(out_path, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
