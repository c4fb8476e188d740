"""ctypes binding of libddfa_b200.so (C ABI declared in include/ddfa_b200.h).

There is NO fallback: if the shared library is missing or a symbol is absent, importing the
binding raises.  Every call checks the status code and raises ``DdfaError`` carrying
``ddfa_last_error()``.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path

from . import build as _build

HEADER = Path(__file__).resolve().parent.parent / "include" / "ddfa_b200.h"

ENGINE_SIMT = 0
ENGINE_TCGEN05 = 1


class DdfaError(RuntimeError):
    pass


def declared_symbols():
    """Function names declared in include/ddfa_b200.h (used by the CPU export test)."""
    text = HEADER.read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ddfa_[a-z0-9_]+)\s*\(", text)))


_vp, _i32, _i64, _f32, _sz = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_size_t
_int = C.c_int

# name -> (restype, argtypes); pointers are passed as integers (tensor.data_ptr()) or ctypes arrays
_SIGNATURES = {
    "ddfa_abi_version": (_int, []),
    "ddfa_last_error": (C.c_char_p, []),
    "ddfa_device_supported": (_int, []),
    "ddfa_launch_count": (C.c_longlong, []),
    "ddfa_engine_available": (_int, [_int]),
    "ddfa_tuning_set": (_int, [_int, _int]),
    "ddfa_tuning_get": (_int, [_int]),
    "ddfa_debug_set": (_int, [_int, _int]),
    "ddfa_debug_read": (_int, [_int, _vp, _sz]),
    "ddfa_build_csr_workspace_bytes": (_sz, [_i64, _i32]),
    "ddfa_build_csr": (_int, [_vp, _vp, _int, _i64, _i32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_graph_ptr": (_int, [_vp, _i32, _vp, _vp]),
    "ddfa_arena_batch_workspace_bytes": (_sz, [_i32]),
    "ddfa_arena_batch": (_int, [_vp, _i32, _i32] + [_vp] * 6 + [_i32, _vp, _i32, _i32] + [_vp] * 7 + [_vp, _sz, _vp]),
    "ddfa_cache_batch_workspace_bytes": (_sz, [_i32]),
    "ddfa_cache_batch": (_int, [_vp, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_embed_concat_fwd": (_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "ddfa_embed_concat_fwd_image": (_int, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "ddfa_embed_concat_bwd": (_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "ddfa_embed_concat_bwd_workspace_bytes": (_sz, [_i32, _i32, _i32, _i32]),
    "ddfa_embed_concat_bwd_ws": (_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _sz, _vp]),
    "ddfa_gather_sum": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _int, _vp]),
    "ddfa_gather_sum_variant": (_int, [_int, _vp, _vp, _vp, _i32, _i32, _vp, _int, _vp]),
    "ddfa_fold_weights_fwd": (_int, [_vp, _vp, _vp, _i32, _vp, _vp, _vp]),
    "ddfa_fold_weights_bwd": (_int, [_vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp]),
    "ddfa_gru_step_workspace_bytes": (_sz, [_i32, _i32, _int]),
    "ddfa_gru_step_prepare": (_int, [_vp] * 5 + [_i32, _int, _vp, _sz, _vp]),
    "ddfa_gru_step_fwd": (_int, [_vp] * 8 + [_i32, _i32, _vp, _vp, _vp, _sz, _int, _vp]),
    "ddfa_act_image_bytes": (_sz, [_i64]),
    "ddfa_act_to_image": (_int, [_vp, _i32, _i32, _vp, _vp]),
    "ddfa_gru_tc_wide_gemm_workspace_bytes": (_sz, [_int, _i32, _i32]),
    "ddfa_gru_tc_wide_gemm": (_int, [_int, _vp, _vp, _i32, _i32, _vp, _vp, _sz, _vp]),
    "ddfa_gru_tc_wide_wgrad_slices": (_sz, [_i32, _i32]),
    "ddfa_gather_sum_image": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "ddfa_gru_step_fwd_image": (_int, [_vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_gather_sum_image_src": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp]),
    "ddfa_gru_gates_packed_bytes": (_sz, [_i32, _i32]),
    "ddfa_gru_step_fwd_image_v2": (_int, [_vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_gru_step_bwd_image_v2": (_int, [_vp] * 9 + [_i32, _i32] + [_vp] * 7 + [_vp, _sz, _int, _vp]),
    "ddfa_gru_step_bwd_image": (_int, [_vp] * 9 + [_i32, _i32] + [_vp] * 7 + [_vp, _sz, _int, _vp]),
    "ddfa_gru_step_bwd_finish": (_int, [_i32, _i32, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_gru_step_bwd_workspace_bytes": (_sz, [_i32, _i32, _int]),
    "ddfa_gru_step_bwd_workspace_bytes_steps": (_sz, [_i32, _i32, _int, _i32]),
    "ddfa_gru_bwd_wgrad_batched": (_int, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_gru_step_prepare_bwd": (_int, [_vp, _vp, _i32, _int, _vp, _sz, _vp]),
    "ddfa_gru_step_bwd": (_int, [_vp] * 7 + [_i32, _i32] + [_vp] * 7 + [_vp, _sz, _int, _vp]),
    "ddfa_ggnn_workspace_bytes": (_sz, [_i32, _i32, _i32, _int, _int]),
    "ddfa_ggnn_fwd": (_int, [_vp, _vp, _vp, _i32, _i32, _i32] + [_vp] * 7 + [_vp, _sz, _int, _int, _vp]),
    "ddfa_ggnn_bwd": (_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32] + [_vp] * 12 + [_vp, _sz, _int, _vp]),
    "ddfa_readout_mlp_fwd": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _i32] + [_vp] * 6 + [_vp]),
    "ddfa_mlp_bwd": (_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "ddfa_readout_bwd": (_int, [_vp] * 5 + [_i32, _i32] + [_vp] * 8 + [_vp]),
    "ddfa_readout_bwd_workspace_bytes": (_sz, [_i32, _i32]),
    "ddfa_readout_bwd_ws": (_int, [_vp] * 5 + [_i32, _i32] + [_vp] * 8 + [_vp, _sz, _vp]),
    "ddfa_graph_label_bce": (_int, [_vp, _vp, _vp, _i32, _f32, _f32, _f32, _vp, _vp, _vp, _vp]),
    "ddfa_graph_label_bce_valid": (_int, [_vp, _vp, _vp, _i32, _i32, _f32, _f32, _f32, _vp, _vp, _vp, _vp]),
    "ddfa_adam_flat": (_int, [_vp, _vp, _vp, _vp, _vp, _i64, _f32, _f32, _f32, _f32, _f32, _vp]),
    "ddfa_allreduce_adam_p2p": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _f32, _f32, _f32, _f32, _f32, _vp]),
    "ddfa_adam_flat_hp": (_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp]),
    "ddfa_allreduce_adam_p2p_hp": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp]),
    "ddfa_grad_norm_workspace_bytes": (_sz, [_i64]),
    "ddfa_grad_norm": (_int, [_vp, _i64, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_adam_flat_guarded": (_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "ddfa_adam_flat_ranges": (_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _vp, _vp, _vp, _vp]),
    "ddfa_p2p_guard_state_bytes": (_sz, []),
    "ddfa_allreduce_adam_p2p_guarded": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "ddfa_adam_flat_groups": (_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _vp, _i32, _vp, _vp, _vp]),
    "ddfa_allreduce_adam_p2p_groups": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i32, _vp, _i32, _vp]),
    "ddfa_allreduce_adam_p2p_groups_guarded": (_int, [_vp, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _i32, _vp, _i32,
                                                      _vp, _vp, _vp, _vp, _vp]),
    "ddfa_node_sample_workspace_bytes": (_sz, [_i32]),
    "ddfa_node_sample": (_int, [_vp, _vp, _i32, C.c_double, C.c_uint64, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_node_head_fwd": (_int, [_vp, _vp, _vp, _vp, _i32, _i32, _vp, _vp, _i32, _vp, _vp, _vp]),
    "ddfa_node_bce": (_int, [_vp, _vp, _vp, _vp, _i32, _f32, _vp, _vp, _vp]),
    "ddfa_node_bce_scaled": (_int, [_vp, _vp, _vp, _vp, _i32, _f32, _f32, _vp, _vp, _vp]),
    "ddfa_node_dp_exchange_words": (_sz, [_i32]),
    "ddfa_node_dp_count": (_int, [_vp, _vp, _i32, C.c_double, _i32, _i32, _vp, _vp, _vp, _sz, _vp, _vp]),
    "ddfa_node_dp_plan": (_int, [_i32, C.c_double, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _sz, _vp, _vp]),
    "ddfa_node_dp_radix_hist": (_int, [_vp, _vp, _i32, C.c_uint64, _i32, _vp, _sz, _vp, _vp]),
    "ddfa_node_dp_radix_pick": (_int, [_i32, _i32, _vp, _sz, _vp, _vp]),
    "ddfa_node_dp_ties": (_int, [_vp, _vp, _i32, C.c_uint64, _i32, _i32, _vp, _sz, _vp, _vp]),
    "ddfa_node_dp_rows": (_int, [_vp, _vp, _i32, C.c_uint64, _i32, _i32, _vp, _vp, _vp, _sz, _vp, _vp]),
    "ddfa_node_bce_global": (_int, [_vp, _vp, _vp, _vp, _vp, _i32, _f32, _f32, _vp, _vp, _vp]),
    "ddfa_node_head_bwd_workspace_bytes": (_sz, [_i32, _i32]),
    "ddfa_node_head_bwd": (_int, [_vp] * 5 + [_i32, _i32, _vp, _i32] + [_vp] * 6 + [_sz, _vp]),
    "ddfa_eval_metrics_workspace_bytes": (_sz, []),
    "ddfa_eval_metrics_graph": (_int, [_vp, _vp, _vp, _i32, _i32, _f32, C.c_double, _vp, _vp, _vp, _i64, _vp, _sz, _vp]),
    "ddfa_eval_metrics_rows": (_int, [_vp, _vp, _vp, _vp, _i32, _f32, C.c_double, _vp, _vp, _vp, _i64, _vp, _sz, _vp]),
    "ddfa_stmt_metric_workspace_bytes": (_sz, []),
    "ddfa_stmt_metric": (_int, [_vp, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp, _sz, _vp]),
    "ddfa_stmt_attention": (_int, [_vp, _vp, _vp, _vp, _i32, _vp, _vp]),
    "ddfa_stmt_input_grad_score": (_int, [_vp, _vp, _vp, _i32, _i32, _i32, _f32, _i32, _vp, _vp]),
    "ddfa_stmt_scale_input": (_int, [_vp, _f32, _i32, _i32, _vp, _vp, _vp]),
    "ddfa_stmt_node_probability": (_int, [_vp, _vp, _i32, _vp, _vp]),
    "ddfa_stmt_attribution_score": (_int, [_vp, _vp, _vp, _i32, _i32, _f32, _i32, _vp, _vp]),
    "ddfa_stmt_shap_input": (_int, [_vp, _vp, _i32, _i32, _i32, _f32, _f32, _f32, C.c_uint64, _vp, _i32, _vp, _vp, _vp, _vp]),
    "ddfa_predict_store": (_int, [_vp, _vp, _vp, _i32, _vp, _i32, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "ddfa_curve_workspace_bytes": (_sz, [_i64]),
    "ddfa_curve_sort": (_int, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_curve_metrics": (_int, [_vp, _vp, _vp, _i64, _vp, _i32] + [_vp] * 10 + [_vp, _sz, _vp]),
    "ddfa_mlp_dgrad_rescale": (_int, [_vp] * 7 + [_i32, _i32, _i32, _vp, _vp, _vp]),
    "ddfa_grad_accumulate": (_int, [_vp, _vp, _i64, _i64, _i32, _vp]),
    "ddfa_csv_index_workspace_bytes": (_sz, [_i64]),
    "ddfa_csv_index_count": (_int, [_vp, _i64, _vp, _vp, _sz, _vp]),
    "ddfa_csv_index_rows": (_int, [_vp, _i64, _vp, _vp, _sz, _vp]),
    "ddfa_csv_fields": (_int, [_vp, _vp, _i64, _vp, _i32, _vp, _vp, _vp]),
    "ddfa_row_sort_workspace_bytes": (_sz, [_i32]),
    "ddfa_row_sort": (_int, [_vp, _i64, _i32, _vp, _i64, _i32, _i32, _vp, _vp, _sz, _vp]),
    "ddfa_csv_graphs_workspace_bytes": (_sz, [_i32]),
    "ddfa_csv_graphs": (_int, [_vp, _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_csv_union": (_int, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _sz] + [_vp] * 6 + [_vp]),
    "ddfa_csv_join_workspace_bytes": (_sz, [_i32]),
    "ddfa_csv_join": (_int, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i32, _vp, _i32, _vp, _vp, _vp, _sz, _vp]),
    "ddfa_sgemm": (_int, [_int, _int, _i32, _i32, _i32, _f32, _vp, _i32, _vp, _i32, _f32, _vp, _i32, _i32, _vp]),
}

TUNE_L2_HINTS, TUNE_PDL_MASK, TUNE_GATHER_VARIANT, TUNE_FWD_PAIR, TUNE_GATE_BWD_TMA, TUNE_GATHER_SRC_GROUPS = 0, 1, 2, 3, 4, 5
TUNE_DETERMINISTIC = 6

_NO_STATUS = {"ddfa_gru_gates_packed_bytes", "ddfa_tuning_get", "ddfa_abi_version", "ddfa_last_error", "ddfa_device_supported", "ddfa_launch_count", "ddfa_engine_available",
              "ddfa_build_csr_workspace_bytes", "ddfa_arena_batch_workspace_bytes", "ddfa_cache_batch_workspace_bytes", "ddfa_gru_step_workspace_bytes", "ddfa_gru_step_bwd_workspace_bytes", "ddfa_gru_step_bwd_workspace_bytes_steps",
              "ddfa_act_image_bytes", "ddfa_ggnn_workspace_bytes", "ddfa_embed_concat_bwd_workspace_bytes", "ddfa_readout_bwd_workspace_bytes",
              "ddfa_grad_norm_workspace_bytes", "ddfa_p2p_guard_state_bytes", "ddfa_node_sample_workspace_bytes",
              "ddfa_node_dp_exchange_words", "ddfa_node_head_bwd_workspace_bytes", "ddfa_eval_metrics_workspace_bytes",
              "ddfa_stmt_metric_workspace_bytes", "ddfa_gru_tc_wide_gemm_workspace_bytes", "ddfa_gru_tc_wide_wgrad_slices",
              "ddfa_curve_workspace_bytes", "ddfa_csv_index_workspace_bytes", "ddfa_row_sort_workspace_bytes",
              "ddfa_csv_graphs_workspace_bytes", "ddfa_csv_join_workspace_bytes"}
EVAL_STATE_WORDS = 16         # DDFA_EVAL_STATE_WORDS: fp64 words of the evaluation metric state
STMT_STATE_WORDS = 16         # DDFA_STMT_STATE_WORDS: fp64 words of the statement metric state
STMT_MODE_VULN_ONLY, STMT_MODE_FULL = 0, 1    # DDFA_STMT_MODE_*: modes of ddfa_stmt_metric
STMT_SCORE_ABS, STMT_SCORE_X_TIMES = 0, 1     # DDFA_STMT_SCORE_*: rules of ddfa_stmt_input_grad_score
CURVE_INFO_WORDS = 8          # DDFA_CURVE_INFO_WORDS: int64 words of the curve info (lengths, class counts, error counts)
PREDICT_MAX_K = 32            # DDFA_PREDICT_MAX_K: the most statements ddfa_predict_store ranks per function
P2P_GUARD_FLAG_WORDS = 96     # DDFA_P2P_GUARD_FLAG_WORDS: flag words per rank the guarded peer-memory exchange needs
GRAD_ACC_SET, GRAD_ACC_ADD, GRAD_ACC_APPLY = 0, 1, 2     # DDFA_GRAD_ACC_*: modes of ddfa_grad_accumulate
ADAM_GROUP_WORDS = 8          # DDFA_ADAM_GROUP_WORDS: fp32 words per row of the parameter-group table
ADAM_MAX_GROUPS = 64          # DDFA_ADAM_MAX_GROUPS: rows the grouped Adam entry points accept
CSV_MAX_COLS = 8              # DDFA_CSV_MAX_COLS: columns one ddfa_csv_fields / ddfa_csv_join call reads or writes
CSV_GRAPH_INFO_WORDS = 8      # DDFA_CSV_GRAPH_INFO_WORDS: int64 words of ddfa_csv_graphs' info
(CSV_ERR_NOT_INT, CSV_ERR_NO_FIELD, CSV_ERR_NO_EDGES, CSV_ERR_NEGATIVE, CSV_ERR_NODE_COUNT, CSV_ERR_NO_FEATURE,
 CSV_ERR_DUPLICATE) = range(1, 8)     # DDFA_CSV_ERR_*: reasons in the error words of the F2 loader


class _Lib:
    def __init__(self):
        path = Path(os.environ["DDFA_LIB_PATH"]) if os.environ.get("DDFA_LIB_PATH") else _build.LIB   # override: A/B of two builds
        if not path.exists():
            raise DdfaError(
                f"{path} is missing: build it with `python -m deepdfa_b200.build` (or __graft_entry__.build()). "
                "deepdfa_b200 has no CPU / PyTorch fallback.")
        self.path = path
        self._dll = C.CDLL(str(path))
        missing = []
        for name, (res, args) in _SIGNATURES.items():
            try:
                fn = getattr(self._dll, name)
            except AttributeError:
                missing.append(name)
                continue
            fn.restype = res
            fn.argtypes = args
        if missing:
            raise DdfaError(f"{path} does not export: {missing}")
        abi = self._dll.ddfa_abi_version()
        if abi != 1:
            raise DdfaError(f"ABI version mismatch: library {abi}, binding 1")
        # A/B scripts select launch configurations through the environment of the PYTHON layer; the library itself reads none
        for env, key in (("DDFA_L2_HINTS", TUNE_L2_HINTS), ("DDFA_PDL", TUNE_PDL_MASK), ("DDFA_GATHER_VARIANT", TUNE_GATHER_VARIANT),
                         ("DDFA_GATE_BWD_TMA", TUNE_GATE_BWD_TMA),
                         ("DDFA_GATHER_SRC_GROUPS", TUNE_GATHER_SRC_GROUPS)):
            if os.environ.get(env) is not None:
                self._dll.ddfa_tuning_set(key, int(os.environ[env]))

    def last_error(self) -> str:
        msg = self._dll.ddfa_last_error()
        return msg.decode() if msg else ""

    def raw(self, name):
        return getattr(self._dll, name)

    def call(self, name, *args):
        rc = getattr(self._dll, name)(*args)
        if name not in _NO_STATUS and rc != 0:
            raise DdfaError(f"{name} failed (status {rc}): {self.last_error()}")
        return rc


_LIB = None


def lib() -> _Lib:
    global _LIB
    if _LIB is None:
        _LIB = _Lib()
    return _LIB


def deterministic_requested() -> bool:
    """The mode the Python layer runs in: DDFA_DETERMINISTIC=0|1 when that is set, else torch.are_deterministic_algorithms_enabled()
    (also True under warn_only=True: every entry point the Python layer calls has a deterministic form, so there is nothing to warn
    about — only C hosts can reach the entry points that refuse the mode)."""
    env = os.environ.get("DDFA_DETERMINISTIC")
    if env is not None:
        if env not in ("0", "1"):
            raise DdfaError(f"DDFA_DETERMINISTIC must be 0 or 1, got {env!r}")
        return env == "1"
    import torch
    return bool(torch.are_deterministic_algorithms_enabled())


def apply_deterministic_mode() -> bool:
    """Sets DDFA_TUNE_DETERMINISTIC to the requested mode (only when it differs from the library's) and returns the mode."""
    want = deterministic_requested()
    L = lib()
    if (L.call("ddfa_tuning_get", TUNE_DETERMINISTIC) == 1) != want:
        L.call("ddfa_tuning_set", TUNE_DETERMINISTIC, int(want))
    return want


def ptr_array(ptrs):
    """Host array of device pointers (for the `const T* const*` parameters)."""
    arr = (C.c_void_p * len(ptrs))(*[C.c_void_p(int(p)) for p in ptrs])
    return arr
