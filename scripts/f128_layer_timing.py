"""Per-layer time of the 3-layer GraphSAGE-T forward, for comparing builds of the F=128 layers (layers 2 and 3): two or
more library builds loaded into ONE process and timed alternately on the benchmark graph (built exactly as bench.py
builds it), the same graph with 64-wide node features (so that layer 1 is an F=64 layer) and the hub-destination and
uniform families, all resident at once.  One round = `--steps` forwards of each
graph with each build in turn, so the builds see the same card, clock and neighbours.

    NERRF_LIB=path/to/parent/libnerrf_b200.so python scripts/f128_layer_timing.py --out DIR [--rounds 5 --steps 5]
    python scripts/f128_layer_timing.py --out DIR --lib parent=A.so --lib this=B.so [--lib other=C.so ...]

Without --lib the builds are the one NERRF_LIB names ("parent") and the in-tree library ("tree").  Writes
DIR/f128_layer_timing.json: per build and graph the median and range of the per-layer and per-forward times (CUDA events
around each layer's launch) and a SHA-256 of the final embeddings and scores (equal digests = the same bits), and the
card's name, power limit, SM clock and clock-throttle reasons read through NVML before and after."""
import argparse
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nerrf_b200 import _lib  # noqa: E402
from nerrf_b200.ai.models import GraphSAGE_T  # noqa: E402
from nerrf_b200.dist import gpu_synthetic_graph  # noqa: E402
from nerrf_b200.graph import synthetic_graph  # noqa: E402

N, E, SEED, F_IN, H, LAYERS = 1_000_000, 10_000_000, 20250115, 32, 128, 3


def card_info():
    import pynvml as nv
    nv.nvmlInit()
    h = nv.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
    name = nv.nvmlDeviceGetName(h)
    return {"name": name.decode() if isinstance(name, bytes) else name,
            "power_limit_w": nv.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
            "sm_clock_mhz": nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM),
            "sm_clock_max_mhz": nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM),
            "throttle_reasons": hex(nv.nvmlDeviceGetCurrentClocksThrottleReasons(h))}


def load(path):
    """ctypes handle of the library at `path` (each path is its own dlopen, with its own CUDA runtime state)."""
    _lib._lib = None
    os.environ["NERRF_LIB"] = path
    return _lib.lib()


def graphs(dev):
    g = synthetic_graph(N, E, seed=SEED)
    out = {"cfg2_hub_src": tuple(torch.from_numpy(a).to(dev) for a in (g.rowptr, g.col, g.ew, g.x))}
    del g
    x64 = torch.randn(N, 64, generator=torch.Generator().manual_seed(SEED)).to(dev)
    out["cfg2_f64_input"] = out["cfg2_hub_src"][:3] + (x64,)
    for fam in ("hub_dst", "uniform"):
        out[fam] = gpu_synthetic_graph(N, E, SEED, dev, family=fam)
    return out


def forward(model, x, rp, col, ew, bufs, score, ev=None):
    inp = x
    if ev: ev[0].record()
    for l in range(LAYERS):
        out = bufs[l & 1]
        model.layer_forward(l, inp, rp, col, ew, out=out, score_out=score if l == LAYERS - 1 else None, reuse_long_scan=l > 0)
        if ev: ev[l + 1].record()
        inp = out
    return inp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH")
    args = ap.parse_args()
    libs = [tuple(s.split("=", 1)) for s in args.lib]
    if not libs:
        if not os.environ.get("NERRF_LIB"):
            sys.exit("set NERRF_LIB to the build to compare against, or pass --lib NAME=PATH at least twice")
        libs = [("parent", os.environ["NERRF_LIB"]), ("tree", _lib.LIB_PATH)]
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    handles = {name: load(os.path.abspath(path)) for name, path in libs}
    models = {F_IN: GraphSAGE_T(F_IN, H, LAYERS).to(dev), 64: GraphSAGE_T(64, H, LAYERS).to(dev)}
    gs = graphs(dev)
    bufs = (torch.empty(N, H, device=dev), torch.empty(N, H, device=dev))
    score = torch.empty(N, device=dev)
    result = {"libraries": {name: os.path.relpath(os.path.abspath(path), ROOT) for name, path in libs},
              "card_before": card_info(), "rounds": args.rounds, "steps": args.steps, "builds": {}}
    digest = {name: {} for name in handles}
    for name, h in handles.items():                                  # warm-up and the digest of the outputs
        _lib._lib = h
        for gname, (rp, col, ew, x) in gs.items():
            for _ in range(3):
                out = forward(models[x.shape[1]], x, rp, col, ew, bufs, score)
            torch.cuda.synchronize()
            d = hashlib.sha256(out.cpu().numpy().tobytes())
            d.update(score.cpu().numpy().tobytes())
            digest[name][gname] = d.hexdigest()
    times = {name: {gname: [] for gname in gs} for name in handles}
    for _ in range(args.rounds):
        for gname, (rp, col, ew, x) in gs.items():
            for name, h in handles.items():
                _lib._lib = h
                evs = [[torch.cuda.Event(enable_timing=True) for _ in range(LAYERS + 1)] for _ in range(args.steps)]
                for s in range(args.steps):
                    forward(models[x.shape[1]], x, rp, col, ew, bufs, score, evs[s])
                torch.cuda.synchronize()
                for ev in evs:
                    times[name][gname].append([ev[l].elapsed_time(ev[l + 1]) for l in range(LAYERS)])
    for name in handles:
        result["builds"][name] = {}
        for gname, tl in times[name].items():
            t = np.array(tl)
            fwd = t.sum(axis=1)
            out = {"output_sha256": digest[name][gname],
                   "forward_ms": {"median": float(np.median(fwd)), "min": float(fwd.min()), "max": float(fwd.max())},
                   "layer_ms_median": [float(m) for m in np.median(t, axis=0)],
                   "layer_ms_min": [float(m) for m in t.min(axis=0)],
                   "layer_ms_max": [float(m) for m in t.max(axis=0)]}
            print(name, gname, json.dumps(out), flush=True)
            result["builds"][name][gname] = out
    for gname in gs:
        same = len({digest[name][gname] for name in handles}) == 1
        print(gname, "same bits in every build" if same else "OUTPUTS DIFFER between builds", flush=True)
    result["card_after"] = card_info()
    with open(os.path.join(args.out, "f128_layer_timing.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["card_before"]), json.dumps(result["card_after"]))


if __name__ == "__main__":
    main()
