"""End-to-end pipeline (trace -> graph -> GNN -> LSTM -> MCTS plan) on a simulator-schema LockBit trace (needs an H100)."""
import numpy as np
import pytest
import torch

from nerrf_b200 import graph as G, pipeline, trace_sim
from nerrf_b200.ai.models import GraphSAGE_T, lstm

pytestmark = pytest.mark.gpu


def test_pipeline_reverts_exactly_the_encrypted_files():
    ev = trace_sim.lockbit_trace(n_files=30, seed=7, benign_files=40)
    g = G.graph_from_events(ev)
    seq, lengths, nodes = pipeline.file_sequences(ev, g)
    assert seq.shape[1:] == (100, 16) and (lengths >= 1).all() and len(nodes) >= 70
    label = g.meta["label"].astype(bool)
    # encrypted files have create + encrypt_start + encrypt_complete events, benign ones only create
    assert set(lengths[np.isin(nodes, np.nonzero(label)[0])]) == {3}
    model = GraphSAGE_T(32, 128, 2).cuda(); seq_model = lstm.LSTMScorer().cuda()
    conf = np.where(label, 0.95, 0.05)            # no trained weights exist (ROADMAP.md M2): labels as confidence
    res = pipeline.run(g, seq, lengths, nodes, model, seq_model, top_a=4096, confidence=conf, n_rollouts=1024,
                       depth=40, iterations=8)
    assert sorted(res.plan_nodes) == sorted(np.nonzero(label)[0].tolist())
    assert res.probs.shape == (len(nodes), 2) and torch.isfinite(res.node_score).all()
    assert set(res.timings_ms) >= {"h2d_graph", "graphsage_t", "lstm", "mcts_plan", "total"}
    # the emitted undo plan renames every encrypted twin back (m1_rollback.sh semantics), in plan order
    from nerrf_b200.ai.planner import emit
    up = emit.from_pipeline(g, res, attack_id="sim-7")
    assert [s["node"] for s in up["steps"]] == res.plan_nodes
    assert all(s["op"] == "rename" and s["from"].endswith(".lockbit3") and s["to"].endswith(".dat") for s in up["steps"])
    assert up["reward_after"] > up["reward_before"]
    # model-driven confidence path runs too (random weights: only structural checks)
    res2 = pipeline.run(g, seq, lengths, nodes, model, seq_model, top_a=32, n_rollouts=256, depth=10, iterations=4, plan_steps=3)
    assert len(res2.candidates) == 32 and len(res2.plan_nodes) <= 3
