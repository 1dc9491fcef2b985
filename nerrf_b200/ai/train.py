"""ai.train -- joint GraphSAGE-T + BiLSTM training (SURVEY.md 8f rank 3).

Reference surface: `ai/train.py` "joint GNN+LSTM training script" (README.md:75 -- named, never written);
gate "GNN / LSTM ROC-AUC >= 0.90 on the toy set" (ROADMAP.md:26,62-69); labels / classes
docs/content/docs/threat-model.mdx:176-203,277-292.

Training is NOT the north-star hot path (that is inference: GraphSAGE_T.forward, lstm.forward, mcts.search,
rewards.score -- CUDA only).  With `--device cuda` the GraphSAGE-T half trains through the library's own kernels: the
fused wgmma layer forward and the hand-written backward (`nerrf_sage_layer_bwd`, csrc/sage_bwd.cu) behind a
torch.autograd.Function (nerrf_b200.ai.autograd); on the CPU it differentiates a plain-torch statement of the same frozen
spec (also the thing the CUDA gradients are tested against).  The BiLSTM half is torch.nn.LSTM under autograd by default;
with `lstm_backward="library"` (`--lstm-backward library`) on a CUDA device it trains through the library's own kernels
instead: the fp32 recurrence saving its activations (`nerrf_lstm_forward_train`) and the backward-through-time of
csrc/lstm_bwd.cu (`nerrf_lstm_backward`), behind nerrf_b200.ai.autograd.LSTMFn.  Both update the very nn.Parameters the CUDA inference kernels read (GraphSAGE_T.weights / biases / node_w /
node_b; LSTMScorer.lstm / head).  Inference never calls anything in this file, and nothing here is a fallback for it:
GraphSAGE_T.forward / LSTMScorer.forward still refuse CPU tensors.

    python -m nerrf_b200.ai.train --traces 8 --epochs 200 --out weights.pt
    python -m nerrf_b200.ai.train --device cuda --fleet 400,8 --bystanders 2 --windows 16 --edge-loss 1.0 --out w.pt
    python -m nerrf_b200.ai.train --device cuda --stream trace.pb --windows 16 --edge-loss 1.0 --out w.pt

The last two train on sliding windows of a trace stream built on the GPU (stream_examples): graph, node and edge labels
and sequences come from the device constructor, so a window can have the size of a fleet window (~10^6 nodes).
"""
from __future__ import annotations

import argparse

import numpy as np
import torch
from torch import nn
from torch.nn.utils.rnn import pack_padded_sequence

from .. import graph as G, pipeline, trace_sim
from .models import GraphSAGE_T
from .models.lstm import LSTMScorer


# ------------------------------------------------------------------ differentiable restatements (autograd only)
def sage_embeddings(model: GraphSAGE_T, x, rowptr, col, ew):
    """Final GraphSAGE-T embeddings with autograd: h' = ReLU([h || m] W + b), m = weighted mean over in-edges (the spec
    in ai/models/graphsage_t.py)."""
    N = x.shape[0]
    deg = (rowptr[1:] - rowptr[:-1]).long()
    dst = torch.repeat_interleave(torch.arange(N, device=x.device), deg)
    src = col.long()
    wsum = torch.zeros(N, device=x.device, dtype=x.dtype).index_add_(0, dst, ew).clamp_min(1e-12)
    h = x
    for W, b in zip(model.weights, model.biases):
        agg = torch.zeros(N, h.shape[1], device=x.device, dtype=x.dtype).index_add_(0, dst, h[src] * ew[:, None])
        h = torch.relu(torch.cat([h, agg / wsum[:, None]], 1) @ W + b)
    return h


def sage_node_logits(model: GraphSAGE_T, x, rowptr, col, ew):
    """Node-head logits of GraphSAGE-T with autograd: logit = h . w_n + b_n over sage_embeddings (sigmoid(logit) is what
    the CUDA forward returns)."""
    return sage_embeddings(model, x, rowptr, col, ew) @ model.node_w + model.node_b


def edge_logits_from_h(model: GraphSAGE_T, h, rowptr, col):
    """Edge-head logits [E, 2] (CSR order; column 0 attack, 1 normal) from embeddings h, with autograd:
    [h_src || h_dst] We + be, computed as (h We[:H])[src] + (h We[H:])[dst] + be (no [E, 2H] intermediate)."""
    H = h.shape[1]
    deg = (rowptr[1:] - rowptr[:-1]).long()
    dst = torch.repeat_interleave(torch.arange(h.shape[0], device=h.device), deg)
    return (h @ model.edge_W[:H])[col.long()] + (h @ model.edge_W[H:])[dst] + model.edge_b


def sage_logits(model: GraphSAGE_T, x, rowptr, col, ew):
    """(node logits [N], edge logits [E, 2]) with autograd: both heads over the same sage_embeddings."""
    h = sage_embeddings(model, x, rowptr, col, ew)
    return h @ model.node_w + model.node_b, edge_logits_from_h(model, h, rowptr, col)


def _train_graph(ex):
    from . import autograd as AG
    tg = ex.get("_train_graph")
    if tg is None:
        tg = ex["_train_graph"] = AG.TrainGraph(ex["rowptr"], ex["col"], ex["ew"])
    return tg


def node_logits(model: GraphSAGE_T, ex):
    """Node-head logits of one example with gradients: on a CUDA device through the library's own kernels (fused wgmma
    forward + csrc/sage_bwd.cu backward, nerrf_b200.ai.autograd), on the CPU through the plain-torch restatement above."""
    if ex["x"].is_cuda:
        from . import autograd as AG
        return AG.sage_node_logits(model, ex["x"], _train_graph(ex))
    return sage_node_logits(model, ex["x"], ex["rowptr"], ex["col"], ex["ew"])


def node_edge_logits(model: GraphSAGE_T, ex):
    """(node logits, edge logits) of one example with gradients: on a CUDA device through the library's kernels (the
    edge head's backward is csrc/sage_edge_bwd.cu), on the CPU through the plain-torch restatement."""
    if ex["x"].is_cuda:
        from . import autograd as AG
        return AG.sage_logits(model, ex["x"], _train_graph(ex))
    return sage_logits(model, ex["x"], ex["rowptr"], ex["col"], ex["ew"])


def edge_loss(edge_logit, edge_label):
    """Class-balanced cross-entropy of the edge head: column 0 = attack (label 1), column 1 = normal (label 0); the
    attack class is weighted by #normal / #attack, clamped to 0.2 .. 5 like the node loss's pos_weight."""
    y = edge_label.to(torch.float32)
    pos = y.sum().clamp_min(1.0)
    w = torch.stack([((y.numel() - pos) / pos).clamp(0.2, 5.0), torch.ones((), device=y.device)])
    return nn.functional.cross_entropy(edge_logit, (1 - edge_label.long()), weight=w)


def lstm_logits(scorer: LSTMScorer, seq, lengths):
    """Head logits [B, 2] of the BiLSTM with autograd (torch.nn.LSTM on packed sequences = the frozen spec)."""
    packed = pack_padded_sequence(seq, lengths.cpu().to(torch.int64), batch_first=True, enforce_sorted=False)
    _, (hn, _) = scorer.lstm(packed)
    return scorer.head(torch.cat([hn[-2], hn[-1]], 1))


def roc_auc(scores, labels) -> float:
    """Area under the ROC curve by the rank statistic (ties get the average rank)."""
    s = np.asarray(scores, np.float64); y = np.asarray(labels).astype(bool)
    n1, n0 = int(y.sum()), int((~y).sum())
    if n1 == 0 or n0 == 0:
        return float("nan")
    order = np.argsort(s, kind="stable")
    ranks = np.empty(s.size, np.float64)
    sorted_s = s[order]
    i = 0
    while i < s.size:
        j = i
        while j + 1 < s.size and sorted_s[j + 1] == sorted_s[i]:
            j += 1
        ranks[order[i:j + 1]] = 0.5 * (i + j) + 1.0
        i = j + 1
    return float((ranks[y].sum() - n1 * (n1 + 1) / 2.0) / (n1 * n0))


# ------------------------------------------------------------------ toy set (simulator-schema LockBit traces)
def make_example(seed: int, n_files: int = 30, benign_files: int = 40, window=None, bystanders: int = 0) -> dict:
    """One labelled example: a simulated LockBit trace -> graph tensors + per-file sequences.  Labels: a file node
    is positive iff it was encrypted (graph.graph_from_events meta['label'], from the simulator's annotations).
    Features are OBSERVABLE-ONLY (graph.OBSERVABLE_SLOT): the annotation event kinds that define the label
    (file_encrypt_start / _complete, ...) are folded onto the syscalls the tracker can actually see
    (openat / write / rename), so the gate below is not satisfied by reading the label back from the input.
    What remains is what a wire trace carries: write / rename counts, byte counts, timing, the .lockbit extension
    ("extension pattern", threat-model.mdx:178-184).  The toy set is still easy; see DESIGN.md 2.7.
    bystanders: benign processes touching the files (trace_sim.lockbit_trace); edge labels: graph meta['edge_label']."""
    ev = trace_sim.lockbit_trace(n_files=n_files, seed=seed, benign_files=benign_files, bystanders=bystanders)
    if window is not None:
        # what the streaming pipeline sees (nerrf_b200.stream): only the events of one sliding window, so a file's
        # history may start with its encryption and the clock features are relative to the window
        t_all = [G._parse_ts(e["timestamp"]) for e in ev]
        lo, hi = t_all[0] + window[0], t_all[0] + window[1]
        ev = [e for e, t_ in zip(ev, t_all) if lo < t_ <= hi]
    g = G.graph_from_events(ev, observable=True, window=None if window is None else float(window[1] - window[0]))
    seq, lengths, nodes = pipeline.file_sequences(ev, g, observable=True)
    t = torch.from_numpy
    return {"x": t(g.x), "rowptr": t(g.rowptr), "col": t(g.col), "ew": t(g.ew),
            "label": t(g.meta["label"].astype(np.float32)), "is_file": t(g.meta["node_kind"] == 0),
            "seq": t(seq), "lengths": t(lengths), "seq_label": t(g.meta["label"][nodes].astype(np.float32)),
            "edge_label": t(g.meta["edge_label"]), "graph": g, "events": ev, "seq_nodes": nodes}


def toy_set(seeds, windows: int = 2, **kw):
    """Per seed: the whole trace plus `windows` random 60 s sliding windows of it (the shape the streamed pipeline feeds
    the models, docs/content/docs/architecture.mdx:39-41)."""
    rng = np.random.default_rng(1234)
    out = []
    for s in seeds:
        nf, nb = int(rng.integers(10, 40)), int(rng.integers(10, 60))
        out.append(make_example(int(s), n_files=nf, benign_files=nb, **kw))
        span = 3.0 + 0.3 * (nf + nb) + 2.0 + 1.41 * nf                # recon + seeding + encryption phases (trace_sim)
        for _ in range(windows):
            hi = float(rng.uniform(0.45, 1.05) * span)
            ex = make_example(int(s), n_files=nf, benign_files=nb, window=(hi - 60.0, hi), **kw)
            if ex["seq"].shape[0] > 1 and 0 < float(ex["label"].sum()):
                out.append(ex)
    return out


# ------------------------------------------------------------------ stream windows (built on the device)
def stream_examples(source, n_windows: int, window_s: float = 60.0, seed: int = 0, files_per_window: int = 512,
                    device="cuda") -> list:
    """`n_windows` labelled examples from random sliding windows of an annotated trace stream, each built on the device:
    the window graph with its node and per-pair edge labels (stream.DeviceStream.window_graph(..., edge_labels=True)),
    and the LSTM sequences (DeviceStream.sequences_device) of a class-balanced sample of at most `files_per_window` file
    nodes -- half encrypted files as far as the window has them, the rest benign.  source: ingest.EventColumns (made
    device resident here, observable-only features like make_example) or a merge-mode stream.DeviceStream.
    Same dict schema as make_example, tensors on the device, so train() / evaluate() take these unchanged; except:
      "events": None (no host event list exists; nothing in train / evaluate reads it),
      "seq" / "lengths" / "seq_label" / "seq_nodes" cover the sampled files only, not every file of the window,
    plus "window": (t_lo, t_hi), the window's bounds in the stream's clock.  Windows with no file node are redrawn."""
    import torch
    from .. import stream
    ds = source if isinstance(source, stream.DeviceStream) else stream.DeviceStream(source, device, observable=True)
    if not ds.merge:
        raise ValueError("stream_examples needs a merge-mode DeviceStream (sequences_device)")
    t_first, t_last = ds.span()
    rng = np.random.default_rng(seed)
    out, draws = [], 0
    while len(out) < n_windows:
        draws += 1
        if draws > 20 * n_windows + 20:
            raise ValueError(f"stream_examples: only {len(out)} of {n_windows} windows hold a file node")
        hi = float(rng.uniform(min(t_first + 0.25 * window_s, t_last), t_last))      # windows end a quarter window in, or later
        g = ds.window_graph(hi - window_s, hi, window_s, edge_labels=True)
        if g is None:
            continue
        lab = g.meta["label"]
        files = np.nonzero(g.meta["node_kind"] == 0)[0]
        if files.size == 0:
            continue
        pos, neg = files[lab[files] > 0], files[lab[files] == 0]
        k_pos = min(pos.size, files_per_window // 2)
        k_neg = min(neg.size, files_per_window - k_pos)
        nodes = np.sort(np.concatenate([rng.choice(pos, k_pos, replace=False), rng.choice(neg, k_neg, replace=False)]))
        seq, lengths = ds.sequences_device(g, nodes)
        dev = g.x.device
        label = torch.from_numpy(lab.astype(np.float32)).to(dev)
        out.append({"x": g.x, "rowptr": g.rowptr, "col": g.col, "ew": g.ew, "label": label,
                    "is_file": torch.from_numpy(g.meta["node_kind"] == 0).to(dev), "seq": seq, "lengths": lengths,
                    "seq_label": label[torch.from_numpy(nodes).to(dev)], "edge_label": g.meta["edge_label"], "graph": g,
                    "events": None, "seq_nodes": nodes, "window": (hi - window_s, hi)})
    return out


def _to(ex, device):
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in ex.items()}


LSTM_BACKWARDS = ("torch", "library")


def train(model: GraphSAGE_T, scorer: LSTMScorer | None, examples, epochs: int = 150, lr: float = 3e-3, device="cpu",
          log=None, lstm_backward: str = "torch", edge_weight: float = 0.0):
    """Joint loss = BCE(node logits over file nodes) + BCE(LSTM encrypt_probability logit); Adam; full batch per trace.
    lstm_backward: "torch" differentiates torch.nn.LSTM (cuDNN on a GPU); "library" runs the BiLSTM forward and
    backward on this library's kernels (nerrf_b200.ai.autograd.lstm_logits) when `device` is a CUDA device.
    edge_weight > 0: the loss also gains edge_weight * the class-balanced cross-entropy of the edge head against
    the examples' edge labels (edge_loss), and the model is marked `edge_head_trained` (a plain attribute, not a
    state_dict entry), which lets pipeline.run attribute files to processes by the edge head."""
    if lstm_backward not in LSTM_BACKWARDS:
        raise ValueError(f"lstm_backward must be one of {LSTM_BACKWARDS}, got {lstm_backward!r}")
    edges = edge_weight > 0
    if edges and model.edge_W is None:
        raise ValueError("edge_weight > 0 needs a model with an edge head")
    device = torch.device(device)
    library_lstm = lstm_backward == "library" and device.type == "cuda"
    if library_lstm:
        from . import autograd as AG
    model.to(device)
    params = list(model.parameters())
    if scorer is not None:
        scorer.to(device)
        params += list(scorer.parameters())
    opt = torch.optim.Adam(params, lr=lr)
    data = [_to(e, device) for e in examples]
    bce = nn.functional.binary_cross_entropy_with_logits
    for ep in range(epochs):
        total = 0.0
        for ex in data:
            opt.zero_grad()
            if edges:
                logit, el = node_edge_logits(model, ex)
            else:
                logit = node_logits(model, ex)
            m = ex["is_file"]
            pos = ex["label"][m].sum().clamp_min(1.0)
            loss = bce(logit[m], ex["label"][m], pos_weight=((m.sum() - pos) / pos).clamp(0.2, 5.0))
            if edges and el.shape[0]:
                loss = loss + edge_weight * edge_loss(el, ex["edge_label"])
            if scorer is not None and ex["seq"].shape[0]:
                if library_lstm:
                    sl = AG.lstm_logits(scorer, ex["seq"], ex["lengths"])
                else:
                    sl = lstm_logits(scorer, ex["seq"], ex["lengths"])
                loss = loss + bce(sl[:, 0], ex["seq_label"]) + 0.5 * bce(sl[:, 1], ex["seq_label"])
            loss.backward()
            opt.step()
            total += float(loss.detach())
        if log and (ep % 25 == 0 or ep == epochs - 1):
            log(f"epoch {ep:4d}  loss {total / len(data):.4f}")
    if edges:
        model.edge_head_trained = True
    return model, scorer


@torch.no_grad()
def evaluate(model: GraphSAGE_T, scorer: LSTMScorer | None, examples, device="cpu", edges: bool = False) -> dict:
    """ROC-AUC of the node scores over file nodes and of the LSTM encrypt_probability over sequences (autograd
    restatement; tests/test_gpu_train.py checks the CUDA inference path gives the same scores).
    edges=True adds edge_auc (P(attack) = softmax column 0 over every labelled edge) and edge_auc_encrypted (only the
    edges incident to an encrypted file: attacker vs. bystander, which the file scores cannot separate)."""
    device = torch.device(device)
    ns, nl, ss, sl_ = [], [], [], []
    es, el_, enc = [], [], []
    for ex in (_to(e, device) for e in examples):
        if edges:
            logit, elog = sage_logits(model.to(device), ex["x"], ex["rowptr"], ex["col"], ex["ew"])
            es.append(torch.softmax(elog, 1)[:, 0].cpu().numpy()); el_.append(ex["edge_label"].cpu().numpy())
            lab = ex["label"].cpu().numpy() > 0
            rp = ex["rowptr"].cpu().numpy().astype(np.int64)
            dst = np.repeat(np.arange(rp.size - 1), np.diff(rp))
            enc.append(lab[ex["col"].cpu().numpy()] | lab[dst])
        else:
            logit = sage_node_logits(model.to(device), ex["x"], ex["rowptr"], ex["col"], ex["ew"])
        m = ex["is_file"]
        ns.append(torch.sigmoid(logit[m]).cpu().numpy()); nl.append(ex["label"][m].cpu().numpy())
        if scorer is not None and ex["seq"].shape[0]:
            p = torch.sigmoid(lstm_logits(scorer.to(device), ex["seq"], ex["lengths"]))
            ss.append(p[:, 0].cpu().numpy()); sl_.append(ex["seq_label"].cpu().numpy())
    out = {"gnn_auc": roc_auc(np.concatenate(ns), np.concatenate(nl))}
    if ss:
        out["lstm_auc"] = roc_auc(np.concatenate(ss), np.concatenate(sl_))
    if edges:
        s, y, e = np.concatenate(es), np.concatenate(el_), np.concatenate(enc)
        out["edge_auc"] = roc_auc(s, y)
        out["edge_auc_encrypted"] = roc_auc(s[e], y[e])
    return out


def _fleet_arg(s: str):
    try:
        procs, attacked = (int(v) for v in s.split(","))
    except ValueError:
        raise argparse.ArgumentTypeError(f"--fleet takes PROCS,ATTACKED (two integers), got {s!r}")
    if not 0 <= attacked <= procs or procs < 1:
        raise argparse.ArgumentTypeError(f"--fleet needs 0 <= ATTACKED <= PROCS and PROCS >= 1, got {s!r}")
    return procs, attacked


def parser() -> argparse.ArgumentParser:
    """The command line of `python -m nerrf_b200.ai.train`."""
    ap = argparse.ArgumentParser(prog="python -m nerrf_b200.ai.train", description=__doc__.split("\n")[0])
    ap.add_argument("--traces", type=int, default=8); ap.add_argument("--epochs", type=int, default=150)
    ap.add_argument("--layers", type=int, default=2); ap.add_argument("--lr", type=float, default=3e-3)
    ap.add_argument("--device", default="cpu"); ap.add_argument("--out", default=None)
    ap.add_argument("--no-lstm", action="store_true")
    ap.add_argument("--lstm-backward", choices=LSTM_BACKWARDS, default="torch",
                    help="BiLSTM training path on a CUDA device: torch.nn.LSTM under autograd, or the library's kernels")
    ap.add_argument("--edge-loss", type=float, default=0.0, metavar="W",
                    help="also train the attack/normal edge head with this loss weight (toy traces get 2 bystander "
                         "processes, so the edge labels differ from the file labels)")
    src = ap.add_mutually_exclusive_group()
    src.add_argument("--fleet", type=_fleet_arg, default=None, metavar="PROCS,ATTACKED",
                     help="train on device-built windows of a simulated fleet trace (stream.fleet_columns, seed --seed) and "
                          "report on windows of a held-out fleet (seed --seed + 1); needs a CUDA device")
    src.add_argument("--stream", default=None, metavar="TRACE_PB",
                     help="train on device-built windows of an annotated EventBatch trace (wire bytes) and report on another "
                          "draw of its windows; needs a CUDA device")
    ap.add_argument("--bystanders", type=int, default=0, metavar="K",
                    help="--fleet: K benign processes per attacked process touching its files after it")
    ap.add_argument("--windows", type=int, default=16, help="--fleet / --stream: training windows")
    ap.add_argument("--window-s", type=float, default=60.0, help="--fleet / --stream: window length in seconds")
    ap.add_argument("--files-per-window", type=int, default=512,
                    help="--fleet / --stream: class-balanced file nodes per window whose sequences train the BiLSTM")
    ap.add_argument("--seed", type=int, default=0, help="--fleet / --stream: fleet seed and window draw")
    return ap


def main(argv=None):
    ap = parser()
    a = ap.parse_args(argv)
    edges = a.edge_loss > 0
    if a.fleet is not None or a.stream is not None:
        if not a.device.startswith("cuda"):
            ap.error("--fleet / --stream build their windows on the GPU: pass --device cuda")
        from .. import ingest, stream
        skw = dict(window_s=a.window_s, files_per_window=a.files_per_window, device=a.device)
        n_test = max(a.windows // 4, 2)
        if a.fleet is not None:
            procs, attacked = a.fleet
            fleet = lambda s: stream.fleet_columns(procs, attacked, seed=s, bystanders=a.bystanders)[0]
            train_set = stream_examples(fleet(a.seed), a.windows, seed=a.seed, **skw)
            test_set = stream_examples(fleet(a.seed + 1), n_test, seed=a.seed + 1, **skw)
        else:
            with open(a.stream, "rb") as f:
                ds = stream.DeviceStream(ingest.decode_event_batch(f.read()), a.device, observable=True)
            train_set = stream_examples(ds, a.windows, seed=a.seed, **skw)
            test_set = stream_examples(ds, n_test, seed=a.seed + 1, **skw)
    else:
        kw = {"bystanders": 2} if edges else {}
        train_set = toy_set(range(100, 100 + a.traces), **kw); test_set = toy_set(range(900, 903), **kw)
    model = GraphSAGE_T(G.F_IN, 128, a.layers); scorer = None if a.no_lstm else LSTMScorer()
    print("before:", evaluate(model, scorer, test_set, a.device, edges=edges))
    train(model, scorer, train_set, a.epochs, a.lr, a.device, log=print, lstm_backward=a.lstm_backward,
          edge_weight=a.edge_loss)
    print("held-out:", evaluate(model, scorer, test_set, a.device, edges=edges))
    if a.out:
        ck = {"sage": model.state_dict(), "lstm": None if scorer is None else scorer.state_dict(), "layers": a.layers}
        if edges:
            ck["edge_head_trained"] = True
        torch.save(ck, a.out)
        print("wrote", a.out)


if __name__ == "__main__":
    main()
