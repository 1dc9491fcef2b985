import numpy as np
import torch

# atol_rms of assert_close_fp32 per GraphSAGE-T layer algo.  "umma2" (2-term bf16 split) is ~1e-5 relative to the tensor
# scale: within the north star's 1e-4 bound but not within the strict absolute floor used for the fp32-equivalent paths.
ATOL_RMS = {"ffma": 1e-5, "umma": 1e-5, "umma2": 1e-4, "auto": 1e-5}


def dev_graph(g, device="cuda", rowptr64=False):
    rp = torch.from_numpy(g.rowptr.astype(np.int64 if rowptr64 else g.rowptr.dtype)).to(device)
    return (torch.from_numpy(g.x).to(device), rp, torch.from_numpy(g.col).to(device), torch.from_numpy(g.ew).to(device))


def cpu_graph(g):
    return (torch.from_numpy(g.x), torch.from_numpy(g.rowptr), torch.from_numpy(g.col), torch.from_numpy(g.ew))


def assert_close_fp32(got, want, rtol=1e-4, atol_rms=1e-5, what=""):
    """The north star's tolerance: embeddings/rewards within 1e-4 relative (fp32).  Elementwise
    |got-want| <= rtol*|want| + atol_rms*rms(want): the absolute term (1e-5 of the tensor's RMS)
    covers entries that are themselves the result of cancellation."""
    got = got.detach().double().cpu(); want = want.detach().double().cpu()
    rms = float(want.pow(2).mean().sqrt()) if want.numel() else 0.0
    err = (got - want).abs()
    tol = rtol * want.abs() + atol_rms * max(rms, 1e-30)
    bad = err > tol
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} out of tolerance, max err {float(err.max()):.3e} (rms {rms:.3e})"
