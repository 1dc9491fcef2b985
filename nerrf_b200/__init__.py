"""nerrf_b200 -- H100-native implementation of the NERRF AI hot path.

GraphSAGE-T temporal scorer, BiLSTM sequence scorer, MCTS rollback planner and reward scorer
(the `ai/` module the reference names in README.md:72-76 but never shipped), as hand-written
sm_90a CUDA behind a C-ABI (include/nerrf_b200.h) with a Python mirror of the reference's
module surface under nerrf_b200.ai (also importable as top-level `ai`).
"""
__version__ = "0.1.0"
