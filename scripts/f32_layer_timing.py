"""Per-layer time of the 3-layer GraphSAGE-T forward, for comparing builds of the F=32 layer (layer 1): the benchmark
graph (built exactly as bench.py builds it) and the hub-destination and uniform families, all resident at once and timed
in interleaved rounds (one round = `--steps` forwards of each graph in turn).

    python scripts/f32_layer_timing.py --out DIR [--rounds 5 --steps 5 --label NAME]

The library timed is the one nerrf_b200 loads (NERRF_LIB selects an experiment build), so two builds are compared by
alternating runs of this script.  Writes DIR/f32_layer_timing[_NAME].json: per graph the median and range of the
per-layer and per-forward times (CUDA events around each layer's launch), a SHA-256 of the final embeddings and scores
(equal digests = the same bits), and the card's name, power limit and SM clock read through NVML before and after."""
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
            "sm_clock_max_mhz": nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)}


def graphs(dev):
    g = synthetic_graph(N, E, seed=SEED)
    out = {"cfg2_hub_src": tuple(torch.from_numpy(a).to(dev) for a in (g.rowptr, g.col, g.ew, g.x))}
    del g
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
    ap.add_argument("--label", default="")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = GraphSAGE_T(F_IN, H, LAYERS).to(dev)
    gs = graphs(dev)
    bufs = (torch.empty(N, H, device=dev), torch.empty(N, H, device=dev))
    score = torch.empty(N, device=dev)
    result = {"library": os.path.relpath(os.environ.get("NERRF_LIB") or _lib.LIB_PATH, ROOT), "card_before": card_info(),
              "rounds": args.rounds, "steps": args.steps, "graphs": {}}
    digest = {}
    for gname, (rp, col, ew, x) in gs.items():                       # warm-up and the digest of the outputs
        for _ in range(3):
            h = forward(model, x, rp, col, ew, bufs, score)
        torch.cuda.synchronize()
        d = hashlib.sha256(h.cpu().numpy().tobytes())
        d.update(score.cpu().numpy().tobytes())
        digest[gname] = d.hexdigest()
    times = {gname: [] for gname in gs}
    for _ in range(args.rounds):
        for gname, (rp, col, ew, x) in gs.items():
            evs = [[torch.cuda.Event(enable_timing=True) for _ in range(LAYERS + 1)] for _ in range(args.steps)]
            for s in range(args.steps):
                forward(model, x, rp, col, ew, bufs, score, evs[s])
            torch.cuda.synchronize()
            for ev in evs:
                times[gname].append([ev[l].elapsed_time(ev[l + 1]) for l in range(LAYERS)])
    for gname, tl in times.items():
        t = np.array(tl)
        fwd = t.sum(axis=1)
        out = {"output_sha256": digest[gname],
               "forward_ms": {"median": float(np.median(fwd)), "min": float(fwd.min()), "max": float(fwd.max())},
               "layer_ms_median": [float(m) for m in np.median(t, axis=0)],
               "layer_ms_min": [float(m) for m in t.min(axis=0)],
               "layer_ms_max": [float(m) for m in t.max(axis=0)]}
        print(gname, json.dumps(out), flush=True)
        result["graphs"][gname] = out
    result["card_after"] = card_info()
    name = "f32_layer_timing" + (f"_{args.label}" if args.label else "") + ".json"
    with open(os.path.join(args.out, name), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["card_after"]))


if __name__ == "__main__":
    main()
