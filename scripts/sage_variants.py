"""Per-layer timing of the fused GraphSAGE-T layer on the three cfg-2-size graph families + a quick cross-check of the
tensor-core path against the fp32 CUDA-core path.  usage: sage_variants.py [reps]"""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200.dist import gpu_synthetic_graph

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
dev = torch.device("cuda", 0)
N, E = 1_000_000, 10_000_000
model = GraphSAGE_T(32, 128, 3).to(dev)
ref = GraphSAGE_T(32, 128, 3, algo="ffma").to(dev)
out = {}
from nerrf_b200.dist import gpu_trace_graph
for fam in ("hub_src", "hub_dst", "uniform", "trace"):
    if fam == "trace":
        rp, col, ew, x, _ = gpu_trace_graph(15625, dev)
        N, E = rp.numel() - 1, col.numel()
    else:
        rp, col, ew, x = gpu_synthetic_graph(N, E, 20250115, dev, family=fam)
    bufs = [torch.empty(N, 128, device=dev) for _ in range(2)]
    score = torch.empty(N, device=dev)
    def step(ev=None):
        inp = x
        for l in range(3):
            if ev: ev[l].record()
            model.layer_forward(l, inp, rp, col, ew, out=bufs[l & 1], score_out=score if l == 2 else None, reuse_long_scan=l > 0)
            inp = bufs[l & 1]
        if ev: ev[3].record()
    for _ in range(3): step()
    torch.cuda.synchronize()
    evs = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(reps)]
    for i in range(reps): step(evs[i])
    torch.cuda.synchronize()
    ms = [sum(evs[i][l].elapsed_time(evs[i][l + 1]) for i in range(reps)) / reps for l in range(3)]
    h_u, s_u = model(x, rp, col, ew)
    h_f, s_f = ref(x, rp, col, ew)
    rms = float(h_f.pow(2).mean().sqrt())
    err = float((h_u - h_f).abs().max()) / rms
    out[fam] = {"layer_ms": ms, "forward_ms": sum(ms), "edges_per_s": E / (sum(ms) * 1e-3), "umma_vs_ffma_max_err_over_rms": err,
                "score_err": float((s_u - s_f).abs().max()), "max_in_degree": int((rp[1:] - rp[:-1]).max())}
    print(fam, json.dumps(out[fam]), flush=True)
    del rp, col, ew, x, bufs
print("RESULT", json.dumps(out))
