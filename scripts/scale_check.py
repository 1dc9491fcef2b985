"""Config-4 size on ONE GPU (10M nodes / 100M edges): size-independent properties of the tensor-core layer.
  (1) W = [0; I], b = 0, x = const  ->  out == const on every non-isolated row, 0 on isolated rows
  (2) random x: 64 sampled rows of out = relu(mean) against an fp64 host evaluation
  (3) full 3-layer forward: finite, deterministic; timing"""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from nerrf_b200 import dist as ND
from nerrf_b200.ai.models import GraphSAGE_T

dev = torch.device("cuda", 0)
N, E = 10_000_000, 100_000_000
t0 = time.time()
rowptr, col, ew, x32 = ND.gpu_synthetic_graph(N, E, 7, dev)
torch.cuda.synchronize(); print(f"graph {N} nodes / {E} edges generated in {time.time() - t0:.1f}s, rowptr {rowptr.dtype}, max deg {int((rowptr[1:] - rowptr[:-1]).max())}")
deg = rowptr[1:] - rowptr[:-1]
model = GraphSAGE_T(128, 128, 1).to(dev)
with torch.no_grad():
    model.weights[0].zero_(); model.weights[0][128:, :] = torch.eye(128, device=dev); model.biases[0].zero_()
x = torch.full((N, 128), 0.75, device=dev)
out = model.layer_forward(0, x, rowptr, col, ew)
nz = deg > 0
print("const test: max |out-0.75| on non-isolated rows %.2e ; isolated rows all zero: %s" % (float((out[nz] - 0.75).abs().max()), bool((out[~nz] == 0).all())))
assert float((out[nz] - 0.75).abs().max()) < 1e-5 and bool((out[~nz] == 0).all())
x = torch.randn(N, 128, device=dev)
out = model.layer_forward(0, x, rowptr, col, ew)
rows = torch.randint(0, N, (64,), device=dev)
worst = 0.0
for r in rows.tolist():
    e0, e1 = int(rowptr[r]), int(rowptr[r + 1])
    if e1 == e0: continue
    w = ew[e0:e1].double(); src = col[e0:e1].long()
    want = torch.relu((x[src].double() * w[:, None]).sum(0) / w.sum())
    worst = max(worst, float((out[r].double() - want).abs().max()))
print("sampled rows vs fp64: max abs err %.2e" % worst)
assert worst < 2e-5
del x, out
m3 = GraphSAGE_T(32, 128, 3).to(dev)
h, sc = m3(x32, rowptr, col, ew)
torch.cuda.synchronize()
e0_ = torch.cuda.Event(enable_timing=True); e1_ = torch.cuda.Event(enable_timing=True)
e0_.record(); h2, sc2 = m3(x32, rowptr, col, ew); e1_.record(); torch.cuda.synchronize()
ms = e0_.elapsed_time(e1_)
print("3-layer forward: %.2f ms = %.2f G edges/s ; finite %s ; deterministic %s" % (ms, E / ms / 1e6, bool(torch.isfinite(h).all()), bool(torch.equal(sc, sc2))))
assert bool(torch.isfinite(h).all()) and bool(torch.equal(sc, sc2)) and bool(torch.equal(h, h2))
print("scale_check ok")
