"""CUDA path against the committed golden fixtures, through the reference-named Python surface (needs an H100)."""
import os

import numpy as np
import pytest
import torch

from ai.models import GraphSAGE_T, lstm
from ai.planner import mcts, rewards
from oracle import sage_ref, lstm_ref
from gpu_util import assert_close_fp32

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_sage_matches_golden():
    gold = np.load(os.path.join(GOLD, "golden_hotpath.npz"))
    model = GraphSAGE_T(32, 128, 2).load_oracle_params(sage_ref.make_params(32, 128, 2, seed=1)).cuda()
    t = lambda k: torch.from_numpy(gold[k]).cuda()
    h, sc, el = model(t("sage_x"), t("sage_rowptr"), t("sage_col"), t("sage_ew"), return_edge_logits=True)
    assert_close_fp32(h, torch.from_numpy(gold["sage_h"]), what="golden h")
    assert_close_fp32(sc, torch.from_numpy(gold["sage_score"]), what="golden score")
    assert_close_fp32(el, torch.from_numpy(gold["sage_edge_logit"]), atol_rms=1e-4, what="golden edge logits")


def test_lstm_matches_golden():
    gold = np.load(os.path.join(GOLD, "golden_hotpath.npz"))
    P = lstm_ref.make_params(16, 256, 2, seed=3)
    model = lstm.LSTMScorer(16, 256, 2)
    model.lstm.load_state_dict(lstm_ref.to_nn_lstm(P, 16, 256).state_dict())
    with torch.no_grad():
        model.head.weight.copy_(P["head_W"]); model.head.bias.copy_(P["head_b"])
    got = model.cuda()(torch.from_numpy(gold["lstm_seq"]).cuda(), torch.from_numpy(gold["lstm_len"]).cuda())
    assert_close_fp32(got, torch.from_numpy(gold["lstm_probs"]), what="golden lstm")


def test_planner_matches_golden_bit_exact():
    gold = np.load(os.path.join(GOLD, "golden_hotpath.npz"))
    act = rewards.Actions(gold["act_p"], gold["act_size"], gold["act_cost"])
    s = rewards.score(gold["rw_states"], act).cpu().numpy()
    assert np.array_equal(s.view(np.uint32), gold["rw_score"].view(np.uint32))
    r = mcts.search(act, rewards.score, n_rollouts=64, depth=10, seed=9, iterations=12)
    assert np.array_equal(r.root_n, gold["mcts_root_n"])
    assert np.array_equal(r.root_w.view(np.uint32), gold["mcts_root_w"].view(np.uint32))
    assert r.best == int(gold["mcts_best"]) and r.num_nodes == int(gold["mcts_num_nodes"])


def test_m1_trace_end_to_end_plan_reverts_the_encrypted_files():
    """cfg 5 in miniature on the reference's own M1 LockBit trace (derived graph fixture): GNN scores are
    computed on the GPU; candidate confidence comes from the trace's attack labels (no trained weights
    exist anywhere -- ROADMAP.md M2), and the plan must revert exactly the 45 files of file_list.txt."""
    tr = np.load(os.path.join(GOLD, "golden_m1_graph.npz"))
    t = lambda k: torch.from_numpy(tr[k]).cuda()
    model = GraphSAGE_T(32, 128, 2).cuda()
    h, sc = model(t("m1_x"), t("m1_rowptr"), t("m1_col"), t("m1_ew"))
    assert torch.isfinite(h).all() and sc.shape[0] == tr["m1_label"].shape[0]
    files = np.nonzero(tr["m1_kind"] == 0)[0]
    label = tr["m1_label"][files].astype(bool)
    act = rewards.Actions(np.where(label, 0.95, 0.05), np.maximum(tr["m1_size_mb"][files], 0.5), np.ones(len(files)))
    pl = mcts.plan(act, max_steps=60, n_rollouts=1024, depth=50, iterations=8)
    assert sorted(files[pl.actions].tolist()) == sorted(np.nonzero(tr["m1_is_listed_encrypted"])[0].tolist())
