"""First hardware check of the tensor-core LSTM path (NERRF_LSTM_ALGO=umma): parity against the oracle, then timing."""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from nerrf_b200.ai.models.lstm import LSTMScorer  # noqa: E402
from oracle import lstm_ref  # noqa: E402


def run(model, seq, ln, algo):
    os.environ["NERRF_LSTM_ALGO"] = algo          # "ffma" = the fp32 CUDA-core cross-check kernel; anything else = wgmma
    out = model(seq, ln)
    torch.cuda.synchronize()
    return out


def main():
    torch.manual_seed(0)
    m = LSTMScorer().cuda()
    for B, T in ((6, 20), (130, 12), (300, 33), (1, 1), (64, 7), (65, 100), (700, 5)):
        seq = torch.randn(B, T, 16); ln = torch.randint(1, T + 1, (B,)); ln[0] = T
        want = lstm_ref.forward(m.oracle_params(), seq, ln)
        for algo in ("ffma", "umma"):
            got = run(m, seq.cuda(), ln.cuda(), algo).cpu()
            print(f"B={B} T={T} {algo}: max err {float((got - want).abs().max()):.3e}", flush=True)
    B, T = 4096, 100
    seq = torch.randn(B, T, 16, device="cuda"); ln = torch.randint(T // 2, T + 1, (B,), device="cuda")
    for algo in ("ffma", "umma"):
        run(m, seq, ln, algo)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a = run(m, seq, ln, algo)
        dt = time.perf_counter() - t0
        print(f"B={B} T={T} {algo}: {dt * 1e3:.2f} ms  {B / dt:.0f} seq/s", flush=True)
        if algo == "ffma":
            ref = a
        else:
            print("umma vs ffma max diff", float((a - ref).abs().max()))


if __name__ == "__main__":
    main()
