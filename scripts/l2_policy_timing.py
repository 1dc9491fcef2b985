"""Per-layer time of the 3-layer GraphSAGE-T forward with the L2 policy of the tensor-core layer off and on
(NERRF_SAGE_FLAG_NO_L2_POLICY, model.l2_policy), interleaved in rounds on the same card, for the benchmark graph (built
exactly as bench.py builds it) and the hub-destination and uniform families.  Also checks that both produce the same bits.

    python scripts/l2_policy_timing.py --out DIR [--rounds 5 --steps 5]

Writes DIR/l2_policy_timing.json: per graph and variant the median and range of the per-layer and per-forward times
(CUDA events around each layer's launches), with the card's name, power limit and SM clock read through NVML."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

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
    yield "cfg2_hub_src", tuple(torch.from_numpy(a).to(dev) for a in (g.rowptr, g.col, g.ew, g.x))
    del g
    for fam in ("hub_dst", "uniform"):
        yield fam, gpu_synthetic_graph(N, E, SEED, dev, family=fam)


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
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = GraphSAGE_T(F_IN, H, LAYERS).to(dev)
    variants = [("off", False), ("on", True)]
    result = {"card_before": card_info(), "rounds": args.rounds, "steps": args.steps, "graphs": {}}
    for gname, (rp, col, ew, x) in graphs(dev):
        bufs = (torch.empty(N, H, device=dev), torch.empty(N, H, device=dev))
        score = torch.empty(N, device=dev)
        times = {v[0]: [] for v in variants}
        ref = None
        same = {}
        for v, on in variants:                                        # warm-up and the bit check
            model.l2_policy = on
            h = forward(model, x, rp, col, ew, bufs, score)
            torch.cuda.synchronize()
            got = (h.clone(), score.clone())
            if ref is None:
                ref = got
            same[v] = bool(torch.equal(got[0].view(torch.int32), ref[0].view(torch.int32)) and
                           torch.equal(got[1].view(torch.int32), ref[1].view(torch.int32)))
        for _ in range(args.rounds):
            for v, on in variants:
                model.l2_policy = on
                evs = [[torch.cuda.Event(enable_timing=True) for _ in range(LAYERS + 1)] for _ in range(args.steps)]
                for s in range(args.steps):
                    forward(model, x, rp, col, ew, bufs, score, evs[s])
                torch.cuda.synchronize()
                for ev in evs:
                    times[v].append([ev[l].elapsed_time(ev[l + 1]) for l in range(LAYERS)])
        out = {}
        for v in times:
            t = np.array(times[v])
            fwd = t.sum(axis=1)
            out[v] = {"same_bits_as_off": same[v],
                      "forward_ms": {"median": float(np.median(fwd)), "min": float(fwd.min()), "max": float(fwd.max())},
                      "layer_ms_median": [float(m) for m in np.median(t, axis=0)],
                      "layer_ms_min": [float(m) for m in t.min(axis=0)],
                      "layer_ms_max": [float(m) for m in t.max(axis=0)]}
            print(gname, v, json.dumps(out[v]), flush=True)
        result["graphs"][gname] = out
        del rp, col, ew, x, bufs, ref
        torch.cuda.empty_cache()
    result["card_after"] = card_info()
    with open(os.path.join(args.out, "l2_policy_timing.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result["card_after"]))


if __name__ == "__main__":
    main()
