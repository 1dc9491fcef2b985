"""Diagnose the tensor-core fused layer against closed-form inputs (run on the GPU box)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from nerrf_b200.ai.models import GraphSAGE_T
from nerrf_b200 import graph as G
from oracle import sage_ref as S

torch.manual_seed(0)
import itertools
for F, algo in itertools.product((32, 128, 64), ("umma", "umma2")):
    print("----", F, algo)
    N = 64 * 3 + 5
    model = GraphSAGE_T(F, 128, 1, algo=algo).cuda()
    W = model.weights[0].detach().cpu(); b = model.biases[0].detach().cpu()
    rp = torch.zeros(N + 1, dtype=torch.int32, device="cuda")
    col = torch.zeros(0, dtype=torch.int32, device="cuda"); ew = torch.zeros(0, device="cuda")
    x = torch.zeros(N, F)
    for r in range(N):
        x[r, r % F] = 1.0
    out = model.layer_forward(0, x.cuda(), rp, col, ew, relu=False).cpu()
    want = W[[r % F for r in range(N)]] + b
    err = (out - want).abs().max().item()
    print(f"[F={F}] one-hot self rows: max err {err:.3e}")
    if err > 1e-4:
        cand = torch.cat([W, torch.zeros(1, 128)]) + b
        for r in list(range(0, 12)) + [63, 64, 65, 130]:
            d = ((cand - out[r]) ** 2).sum(1)
            k = int(d.argmin())
            print(f"   row {r}: expected k={r % F}, best match k={k} (dist {float(d[k]):.2e}); out[:4]={out[r,:4].tolist()} want[:4]={want[r,:4].tolist()}")
    # random dense rows, no edges: tests the hi/lo split accuracy
    x = torch.randn(N, F)
    out = model.layer_forward(0, x.cuda(), rp, col, ew, relu=False).cpu()
    want = torch.cat([x, torch.zeros(N, F)], 1).double() @ W.double() + b.double()
    rel = ((out.double() - want).abs() / (want.abs() + 1e-3 * want.abs().mean())).max().item()
    print(f"[F={F}] random self rows vs fp64: max rel err {rel:.3e}")
    # with edges
    g = G.synthetic_graph(N=1000, E=12000, seed=3, f_in=F)
    t = lambda a: torch.from_numpy(a)
    out = model.layer_forward(0, t(g.x).cuda(), t(g.rowptr).cuda(), t(g.col).cuda(), t(g.ew).cuda()).cpu()
    want = S.layer(t(g.x), t(g.rowptr), t(g.col), t(g.ew), W, b, dtype=torch.float64)
    err = (out.double() - want).abs()
    print(f"[F={F}] graph layer vs fp64 oracle: max abs err {err.max().item():.3e}, rms {want.pow(2).mean().sqrt().item():.3e}")
print("umma_debug done")
