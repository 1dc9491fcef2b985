"""ctypes binding of the C-ABI library (include/nerrf_b200.h).

The product path has NO CPU fallback: if the shared library is missing or a call fails this
module raises.  It never imports anything from ``oracle/``.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libnerrf_b200.so")

_lib = None

i32p = C.POINTER(C.c_int32)
u32p = C.POINTER(C.c_uint32)
f32p = C.POINTER(C.c_float)
vp = C.c_void_p

# name -> (restype, argtypes); mirrors include/nerrf_b200.h one to one
SIGNATURES = {
    "nerrf_abi_version": (C.c_int, []),
    "nerrf_last_error": (C.c_char_p, []),
    "nerrf_device_info": (C.c_int, [i32p, i32p, i32p]),
    "nerrf_sage_aggregate": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, C.c_int64, C.c_int64, C.c_int64, C.c_int, vp]),
    "nerrf_sage_layer_fwd": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp, vp, C.c_int64, C.c_int64, C.c_int64,
                                       C.c_int, C.c_int, C.c_int, C.c_int, vp]),
    "nerrf_sage_layer_head_fwd": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp, vp, C.c_int64, C.c_int64, C.c_int64,
                                            C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_float, vp, vp]),
    "nerrf_sage_layer_bwd_workspace_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "nerrf_sage_layer_bwd": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_size_t, C.c_int64, C.c_int,
                                       C.c_int, C.c_int, vp]),
    "nerrf_sage_norm_weights": (C.c_int, [vp, C.c_int, vp, vp, C.c_int64, vp]),
    "nerrf_sage_layer_bwd_ex": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_size_t, C.c_int64,
                                          C.c_int, C.c_int, C.c_int, vp, C.c_int, vp, vp, vp, vp]),
    "nerrf_explain_subgraph_workspace_bytes": (C.c_int, [C.c_int64, C.c_int64, C.POINTER(C.c_size_t)]),
    "nerrf_explain_subgraph_count": (C.c_int, [vp, C.c_int, vp, C.c_int64, vp, C.c_int64, C.c_int, C.c_int64, vp, vp,
                                               C.c_size_t, vp]),
    "nerrf_explain_subgraph_fill": (C.c_int, [vp, C.c_int, vp, vp, vp, C.c_int, C.c_int64, vp, C.c_int64, C.c_int, C.c_int64,
                                              vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "nerrf_explain_topk": (C.c_int, [vp, C.c_int64, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]),
    "nerrf_lstm_explain_steps": (C.c_int, [vp, vp, vp, C.c_int64, C.c_int, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp]),
    "nerrf_incident_files_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_size_t)]),
    "nerrf_incident_files": (C.c_int, [vp, C.c_int, vp, C.c_int64, vp, vp, C.c_float, vp, C.c_int64, vp, vp, vp, vp, vp, vp,
                                       C.POINTER(C.c_int64), vp, C.c_size_t, vp]),
    "nerrf_incident_group_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_size_t)]),
    "nerrf_incident_group": (C.c_int, [vp, vp, vp, C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "nerrf_taint_closure_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_size_t)]),
    "nerrf_taint_closure": (C.c_int, [vp, C.c_int, vp, C.c_int64, vp, vp, vp, vp, vp, vp, C.c_int64, C.c_int, vp, vp, vp, vp, vp,
                                      C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int32), vp, vp, C.c_size_t, vp]),
    "nerrf_trace_flow_class": (C.c_int, [vp, vp, vp, C.c_int64, vp]),
    "nerrf_trace_flow_class_device": (C.c_int, [vp, vp, vp, C.c_int64, vp, vp]),
    "nerrf_sage_edge_head_bwd_workspace_bytes": (C.c_int, [C.c_int64, C.c_int, C.POINTER(C.c_size_t)]),
    "nerrf_sage_edge_head_bwd": (C.c_int, [vp, vp, vp, vp, C.c_int, vp, vp, C.c_int, vp, vp, vp, vp, C.c_size_t,
                                           C.c_int64, C.c_int, vp]),
    "nerrf_sage_long_rows_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_size_t)]),
    "nerrf_sage_layer_fwd_ex": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp, vp, C.c_int64, C.c_int64, C.c_int64,
                                          C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_float, vp, vp, C.c_size_t,
                                          C.POINTER(vp), C.c_int, vp, vp]),
    "nerrf_sage_node_head": (C.c_int, [vp, vp, C.c_float, vp, vp, vp, C.c_int64, C.c_int64, C.c_int, vp]),
    "nerrf_sage_edge_head": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, C.c_int64, C.c_int64, vp]),
    "nerrf_sage_forward": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int64, C.c_int, C.c_int, C.c_int,
                                     C.POINTER(vp), C.POINTER(vp), vp, C.c_float, vp, vp, vp, C.c_size_t, C.c_int, vp]),
    "nerrf_sage_session_create": (C.c_int, [C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "nerrf_sage_session_set_weights": (C.c_int, [vp, C.POINTER(vp), C.POINTER(vp), vp, C.c_float]),
    "nerrf_sage_session_forward_host": (C.c_int, [vp, vp, vp, vp, vp, C.c_int64, C.c_int64, vp, vp, C.c_int]),
    "nerrf_sage_session_submit_host": (C.c_int, [vp, vp, vp, vp, vp, C.c_int64, C.c_int64, vp, vp, C.c_int, C.POINTER(C.c_uint64)]),
    "nerrf_sage_session_wait": (C.c_int, [vp, C.c_uint64]),
    "nerrf_sage_session_destroy": (C.c_int, [vp]),
    "nerrf_reward_score": (C.c_int, [vp, C.c_int64, vp, vp, vp, vp, C.c_int, vp, vp]),
    "nerrf_mcts_workspace_bytes": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "nerrf_mcts_search": (C.c_int, [vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_float,
                                    C.c_float, C.c_float, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "nerrf_mcts_search_host": (C.c_int, [vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_float,
                                         C.c_float, C.c_float, vp, vp, vp, vp]),
    "nerrf_plan_commit_workspace_bytes": (C.c_int, [C.c_int, C.POINTER(C.c_size_t)]),
    "nerrf_plan_commit": (C.c_int, [vp, vp, vp, vp, C.c_int, vp, vp, C.c_int, C.c_float, C.c_int, C.c_int, vp, vp, vp, vp, C.c_size_t, vp]),
    "nerrf_mcts_session_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(vp)]),
    "nerrf_mcts_session_search_host": (C.c_int, [vp, vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_uint64,
                                                 C.c_float, C.c_float, C.c_float, vp, vp, vp, vp]),
    "nerrf_mcts_session_destroy": (C.c_int, [vp]),
    "nerrf_reward_score_ex": (C.c_int, [vp, C.c_int64, vp, vp, vp, vp, vp, C.c_int, vp, vp]),
    "nerrf_mcts_search_ex": (C.c_int, [vp, vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_float,
                                       C.c_float, C.c_float, vp, vp, vp, vp, vp, C.c_size_t, vp]),
    "nerrf_mcts_search_host_ex": (C.c_int, [vp, vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_float,
                                            C.c_float, C.c_float, vp, vp, vp, vp]),
    "nerrf_plan_commit_ex": (C.c_int, [vp, vp, vp, vp, vp, C.c_int, vp, vp, C.c_int, C.c_float, C.c_int, C.c_int, vp, vp, vp, vp,
                                       C.c_size_t, vp]),
    "nerrf_mcts_session_search_host_ex": (C.c_int, [vp, vp, vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_uint64,
                                                    C.c_float, C.c_float, C.c_float, vp, vp, vp, vp]),
    "nerrf_lstm_workspace_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "nerrf_lstm_forward": (C.c_int, [vp, vp, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp),
                                     C.POINTER(vp), C.POINTER(vp), vp, vp, vp, vp, C.c_size_t, vp]),
    "nerrf_lstm_train_workspace_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t),
                                                   C.POINTER(C.c_size_t)]),
    "nerrf_lstm_forward_train": (C.c_int, [vp, vp, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp),
                                           C.POINTER(vp), C.POINTER(vp), vp, vp, C.c_size_t, vp]),
    "nerrf_lstm_backward": (C.c_int, [vp, vp, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp), C.POINTER(vp),
                                      vp, C.c_size_t, vp, vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), vp, C.c_size_t,
                                      vp]),
    "nerrf_lstm_input_grad_workspace_bytes": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_size_t)]),
    "nerrf_lstm_input_grad": (C.c_int, [vp, vp, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(vp), C.POINTER(vp),
                                        vp, C.c_size_t, vp, vp, vp, C.c_size_t, vp]),
    "nerrf_graph_csr_workspace_bytes": (C.c_int, [C.c_int64, C.c_int64, C.POINTER(C.c_int64)]),
    "nerrf_graph_build_csr_ex": (C.c_int, [vp, vp, vp, vp, C.c_int64, C.c_int64, C.c_float, C.c_float, vp, C.c_int,
                                           vp, vp, vp, vp, C.c_int64, vp]),
    "nerrf_trace_sequences": (C.c_int, [vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_double, C.c_double, C.c_int, vp, vp, vp]),
    "nerrf_trace_sequences_ex": (C.c_int, [vp, C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_double, C.c_double, C.c_int, vp, vp,
                                           vp, vp]),
    "nerrf_graph_build_csr": (C.c_int, [vp, vp, vp, vp, C.c_int64, C.c_int64, C.c_float, C.c_float, vp, C.c_int,
                                        vp, vp, vp, C.c_int64, vp]),
    "nerrf_trace_edge_labels_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_int64)]),
    "nerrf_trace_edge_labels": (C.c_int, [vp, vp, vp, C.c_int64, vp, C.c_int, vp, C.c_int64, C.c_int64, vp, vp, C.c_int64, vp]),
    "nerrf_graph_node_features_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_int64)]),
    "nerrf_graph_node_features": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.c_int64, vp, C.c_int64, C.c_double, vp, vp, vp,
                                            vp, C.c_int64, vp]),
    "nerrf_trace_scan": (C.c_int, [vp, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "nerrf_trace_decode": (C.c_int, [vp, C.c_int64, C.c_int64] + [vp] * 17),
    "nerrf_trace_path_flags": (C.c_int, [vp, vp, C.c_int64, vp]),
    "nerrf_trace_frame": (C.c_int, [vp, C.c_int64, C.c_int, C.c_int64, vp, vp, vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "nerrf_trace_decode_device_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_int64)]),
    "nerrf_trace_decode_device": (C.c_int, [vp, vp, vp, vp, C.c_int64, C.c_int64, C.POINTER(vp), vp, vp, C.c_int64, vp]),
    "nerrf_trace_stream_order_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_int64)]),
    "nerrf_trace_stream_order": (C.c_int, [C.c_int64, vp, vp, vp, vp, C.c_double, vp, vp, vp, vp, vp, vp, C.POINTER(C.c_int64),
                                           vp, C.c_int64, vp]),
    "nerrf_trace_stream_columns": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, vp, vp]),
    "nerrf_trace_gather_rows_workspace_bytes": (C.c_int, [C.c_int64, C.POINTER(C.c_int64)]),
    "nerrf_trace_gather_rows": (C.c_int, [C.POINTER(vp), vp, C.c_int64, C.POINTER(vp), vp, C.c_int64, vp]),
    "nerrf_trace_intern_device_workspace_bytes":(C.c_int, [C.c_int64, C.c_int64, C.POINTER(C.c_int64)]),
    "nerrf_trace_intern_device": (C.c_int, [C.c_int64, C.c_int64, vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, C.POINTER(C.c_int64),
                                            vp, vp, vp, C.c_int64, vp, C.c_int64, vp]),
    "nerrf_trace_name_hash": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "nerrf_trace_dir_hash": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "nerrf_trace_intern": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, C.POINTER(C.c_int64),
                                     vp, vp, vp, C.c_int64]),
    "nerrf_trace_decode_device_ex": (C.c_int, [vp, vp, vp, vp, C.c_int64, C.c_int64, C.POINTER(vp), vp, C.c_int, vp, vp, C.c_int64,
                                               vp]),
    "nerrf_trace_stream_order_ex": (C.c_int, [C.c_int64, vp, vp, vp, vp, C.c_int, vp, C.c_double, vp, vp, vp, vp, vp, vp,
                                              C.POINTER(C.c_int64), vp, C.c_int64, vp]),
    "nerrf_trace_gather_rows_ex": (C.c_int, [C.POINTER(vp), vp, vp, C.c_int64, C.POINTER(vp), vp, vp, C.c_int64, vp]),
    "nerrf_trace_intern_device_ex": (C.c_int, [C.c_int64, C.c_int64, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp,
                                               C.POINTER(C.c_int64), vp, vp, vp, C.c_int64, vp, C.c_int64, vp]),
    "nerrf_trace_name_hash_ex": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "nerrf_trace_dir_hash_ex": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "nerrf_trace_intern_ex": (C.c_int, [C.c_int64, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp, C.POINTER(C.c_int64),
                                        vp, vp, vp, C.c_int64]),
}


class NerrfError(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle.  Raises if the library was not built."""
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("NERRF_LIB") or LIB_PATH                 # experiment builds of the same library (scripts/)
    if not os.path.exists(path):
        raise NerrfError(
            f"{path} not found: build it with `python -m nerrf_b200.build` "
            "(nvcc, sm_90a).  There is no CPU fallback.")
    h = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(h, name)          # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if h.nerrf_abi_version() != 2:
        raise NerrfError("ABI version mismatch between nerrf_b200/_lib.py and libnerrf_b200.so")
    _lib = h
    return h


def check(rc, what=""):
    if rc != 0:
        msg = lib().nerrf_last_error()
        raise NerrfError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")


def ptr(t):
    """Device/host pointer of a torch tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def ptr_array(tensors):
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


def current_stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise NerrfError("nerrf_b200 kernels need CUDA tensors (no CPU fallback); got a CPU tensor")
