"""`python -m nerrf_b200.undo`: EventBatch wire file in, undo plan out (needs an H100)."""
import json

import pytest

from nerrf_b200 import ingest, trace_sim, undo

pytestmark = pytest.mark.gpu


def test_undo_cli_from_wire_bytes(tmp_path):
    ev = trace_sim.lockbit_trace(n_files=18, seed=21, benign_files=25)
    (tmp_path / "events.pb").write_bytes(ingest.encode_event_batch(ev))
    out, sh = tmp_path / "plan.json", tmp_path / "plan.sh"
    plan = undo.main(["--trace", str(tmp_path / "events.pb"), "--train-epochs", "25", "--out", str(out), "--shell", str(sh),
                      "--id", "sim-21", "--rollouts", "512", "--depth", "30", "--iterations", "6"])
    assert json.loads(out.read_text()) == plan and plan["attack_id"] == "sim-21"
    renamed = sorted(s["from"] for s in plan["steps"])
    encrypted = sorted({e["path"] for e in ev if e["path"].endswith(".lockbit3")})
    assert renamed == encrypted and len(encrypted) == 18
    assert all(s["op"] == "rename" for s in plan["steps"]) and plan["reward_after"] > plan["reward_before"]
    assert sh.read_text().count("mv -- ") == 18
    assert plan["stats"]["events"] == len(ev) and plan["stats"]["nodes"] > 40


def test_undo_cli_needs_weights(tmp_path):
    (tmp_path / "e.pb").write_bytes(ingest.encode_event_batch(trace_sim.lockbit_trace(n_files=3, seed=1)))
    with pytest.raises(SystemExit, match="no weights"):
        undo.main(["--trace", str(tmp_path / "e.pb")])
