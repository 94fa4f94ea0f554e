"""Loads ``libctc_crf_b200.so`` and declares the C ABI of ``include/ctc_crf_b200.h`` for ctypes.

There is no fallback: if the library is missing the import fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

from .build import LIB

_lib = None


class ctcOptions(C.Structure):
    """gpu_ctc/ctc.h:36-39"""
    _fields_ = [("stream", C.c_void_p), ("blank_label", C.c_int)]


# every symbol include/ctc_crf_b200.h declares (tests check the export list against the header)
SYMBOLS = [
    "Init", "Release", "compute_alpha", "compute_beta_and_grad", "compute_ctc_loss", "get_workspace_size",
    "ctcGetStatusString", "ccb_last_error", "ccb_den_loaded", "ccb_den_info", "ccb_den_alpha_floats", "ccb_den_aux_bytes",
    "ccb_ctc_workspace_bytes", "ccb_den_forward_backward", "ccb_ctc_forward_backward", "ccb_ctc_crf_loss_fwd",
    "ccb_ctc_crf_loss_logits_fwd", "ccb_ctc_loss_fwd", "ccb_ctc_align_workspace_bytes", "ccb_ctc_align",
    "ccb_launch_count", "ccb_debug_timeline", "ccb_plan_create", "ccb_plan_destroy", "ccb_plan_info", "ccb_plan_copy",
    "ccb_plan_launch", "ccb_plan_launch_own",
    "ccb_den_ckpt_alpha_floats", "ccb_ctc_crf_loss_ckpt_fwd", "ccb_ctc_crf_loss_logits_ckpt_fwd",
    "ccb_den_fwd_alpha_floats", "ccb_num_fwd_only_bytes", "ccb_ctc_crf_loss_fwd_only", "ccb_ctc_loss_fwd_only",
    "ccb_ctc_crf_loss_costs", "ccb_ctc_crf_loss_costs_fwd_only", "ccb_ctc_loss_costs", "ccb_grad_rows_scale",
    "ccb_ctc_crf_loss_seqs", "ccb_ctc_crf_loss_seqs_fwd_only", "ccb_ctc_loss_seqs", "ccb_seqs_grad", "ccb_ctc_align_seqs",
    "ccb_crf_sample_ws_bytes", "ccb_crf_sample", "ccb_ctc_beam_search_ws_bytes", "ccb_ctc_beam_search", "ccb_plan_ctc_shape",
    "ccb_ngram_create", "ccb_ngram_destroy", "ccb_ngram_info", "ccb_ngram_copy", "ccb_ctc_beam_search_lm",
    "ccb_wfst_create", "ccb_wfst_destroy", "ccb_wfst_info", "ccb_wfst_copy", "ccb_wfst_decode_ws_bytes", "ccb_wfst_decode",
    "ccb_rnnt_workspace_bytes", "ccb_rnnt_forward", "ccb_rnnt_backward", "ccb_gather_ws_bytes", "ccb_gather_sum",
    "ccb_gather_sum_backward", "ccb_rnnt_simple_workspace_bytes", "ccb_rnnt_simple_forward", "ccb_rnnt_simple_backward",
    "ccb_ctct_workspace_bytes", "ccb_ctct_forward", "ccb_ctct_backward", "ccb_ctct_simple_workspace_bytes",
    "ccb_ctct_simple_forward", "ccb_ctct_simple_backward", "ccb_rnnt_beam_ws_bytes", "ccb_rnnt_beam_init",
    "ccb_rnnt_beam_step", "ccb_rnnt_beam_finish", "ccb_ctct_beam_ws_bytes", "ccb_ctct_beam_init", "ccb_ctct_beam_step",
    "ccb_rnnt_beam_step_fused", "ccb_ngram_slot_rows", "ccb_lm_mix_slot_rows", "ccb_ngram_score",
]
GLOBALS = ["DEN_NUM_ARCS", "DEN_NUM_STATES"]


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB):
        raise ImportError(
            f"{LIB} is missing: build it with `python -m cat_b200.build` (nvcc, sm_90a). "
            "cat_b200 has no CPU or PyTorch fallback.")
    L = C.CDLL(LIB)
    vp, ip, fp = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_float)
    L.Init.argtypes = [C.c_char_p, C.c_int, ip]; L.Init.restype = None
    L.Release.argtypes = [C.c_int, ip]; L.Release.restype = None
    L.compute_alpha.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    L.compute_alpha.restype = None
    L.compute_beta_and_grad.argtypes = [vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp]
    L.compute_beta_and_grad.restype = None
    L.compute_ctc_loss.argtypes = [vp, vp, ip, ip, ip, C.c_int, C.c_int, fp, vp, ctcOptions]
    L.compute_ctc_loss.restype = C.c_int
    L.get_workspace_size.argtypes = [ip, ip, C.c_int, C.c_int, ctcOptions, C.POINTER(C.c_size_t)]
    L.get_workspace_size.restype = C.c_int
    L.ctcGetStatusString.argtypes = [C.c_int]; L.ctcGetStatusString.restype = C.c_char_p
    L.ccb_last_error.argtypes = []; L.ccb_last_error.restype = C.c_char_p
    L.ccb_den_loaded.argtypes = [C.c_int]; L.ccb_den_loaded.restype = C.c_int
    L.ccb_den_info.argtypes = [C.POINTER(C.c_long)]; L.ccb_den_info.restype = C.c_int
    L.ccb_den_alpha_floats.argtypes = [C.c_int, C.c_int]; L.ccb_den_alpha_floats.restype = C.c_size_t
    L.ccb_den_aux_bytes.argtypes = [C.c_int, C.c_int]; L.ccb_den_aux_bytes.restype = C.c_size_t
    L.ccb_ctc_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]; L.ccb_ctc_workspace_bytes.restype = C.c_size_t
    L.ccb_den_forward_backward.argtypes = [vp, C.c_int, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int, vp, vp, vp,
                                           vp, C.c_long, C.c_long, C.c_float, vp, vp, vp]
    L.ccb_den_forward_backward.restype = C.c_int
    L.ccb_ctc_forward_backward.argtypes = [vp, C.c_int, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp,
                                           C.c_int, C.c_int, vp, vp, C.c_long, C.c_long, C.c_float, vp, vp]
    L.ccb_ctc_forward_backward.restype = C.c_int
    L.ccb_ctc_crf_loss_fwd.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int,
                                       C.c_float, C.c_float, vp, vp, vp, vp, vp, vp, vp]
    L.ccb_ctc_crf_loss_fwd.restype = C.c_int
    L.ccb_ctc_crf_loss_logits_fwd.argtypes = L.ccb_ctc_crf_loss_fwd.argtypes
    L.ccb_ctc_crf_loss_logits_fwd.restype = C.c_int
    L.ccb_den_ckpt_alpha_floats.argtypes = [C.c_int, C.c_int, C.c_int]; L.ccb_den_ckpt_alpha_floats.restype = C.c_size_t
    L.ccb_ctc_crf_loss_ckpt_fwd.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int,
                                            C.c_float, C.c_float, vp, vp, vp, vp, vp, vp, vp]
    L.ccb_ctc_crf_loss_ckpt_fwd.restype = C.c_int
    L.ccb_ctc_crf_loss_logits_ckpt_fwd.argtypes = L.ccb_ctc_crf_loss_ckpt_fwd.argtypes
    L.ccb_ctc_crf_loss_logits_ckpt_fwd.restype = C.c_int
    L.ccb_ctc_loss_fwd.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int,
                                   C.c_float, vp, vp, vp, vp, vp]
    L.ccb_ctc_loss_fwd.restype = C.c_int
    L.ccb_den_fwd_alpha_floats.argtypes = [C.c_int]; L.ccb_den_fwd_alpha_floats.restype = C.c_size_t
    L.ccb_num_fwd_only_bytes.argtypes = [C.c_int]; L.ccb_num_fwd_only_bytes.restype = C.c_size_t
    L.ccb_ctc_crf_loss_fwd_only.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int,
                                            C.c_float, C.c_float, vp, vp, vp, vp, vp, vp]
    L.ccb_ctc_crf_loss_fwd_only.restype = C.c_int
    L.ccb_ctc_loss_fwd_only.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int,
                                        C.c_float, vp, vp, vp]
    L.ccb_ctc_loss_fwd_only.restype = C.c_int
    L.ccb_ctc_crf_loss_costs.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp,
                                         C.c_int, C.c_float, C.c_float, vp, vp, vp, vp, vp, vp, vp, C.c_int, vp]
    L.ccb_ctc_crf_loss_costs.restype = C.c_int
    L.ccb_ctc_crf_loss_costs_fwd_only.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp,
                                                  C.c_int, C.c_float, C.c_float, vp, vp, vp, vp, vp, vp, C.c_int, vp]
    L.ccb_ctc_crf_loss_costs_fwd_only.restype = C.c_int
    L.ccb_ctc_loss_costs.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int,
                                     C.c_float, vp, vp, vp, vp, vp, C.c_int, vp]
    L.ccb_ctc_loss_costs.restype = C.c_int
    L.ccb_grad_rows_scale.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]
    L.ccb_grad_rows_scale.restype = C.c_int
    L.ccb_ctc_align_workspace_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
    L.ccb_ctc_align_workspace_bytes.restype = C.c_size_t
    L.ccb_ctc_align.argtypes = [vp, C.c_int, C.c_long, C.c_long, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int,
                                vp, vp, vp, vp]
    L.ccb_ctc_align.restype = C.c_int
    i, f, l = C.c_int, C.c_float, C.c_long
    L.ccb_ctc_crf_loss_seqs.argtypes = [vp, i, i, i, i, i, i, i, vp, vp, vp, vp, i, vp, vp, vp, i, f, f, vp, vp, vp, vp, vp,
                                        vp, i, i, vp]
    L.ccb_ctc_crf_loss_seqs.restype = C.c_int
    L.ccb_ctc_crf_loss_seqs_fwd_only.argtypes = [vp, i, i, i, i, i, i, vp, vp, vp, vp, i, vp, vp, i, f, f, vp, vp, vp, vp,
                                                 vp, i, vp]
    L.ccb_ctc_crf_loss_seqs_fwd_only.restype = C.c_int
    L.ccb_ctc_loss_seqs.argtypes = [vp, i, i, i, i, i, vp, vp, vp, vp, i, vp, vp, vp, i, i, f, vp, vp, vp, vp, vp, i, i, vp]
    L.ccb_ctc_loss_seqs.restype = C.c_int
    L.ccb_seqs_grad.argtypes = [vp, i, i, i, i, i, i, vp, vp, vp, vp, i, vp, vp, i, i, f, vp, vp, vp, vp, i, vp, vp]
    L.ccb_seqs_grad.restype = C.c_int
    L.ccb_ctc_align_seqs.argtypes = [vp, i, l, l, i, i, i, vp, vp, vp, vp, i, vp, vp, i, i, vp, vp, vp, vp]
    L.ccb_ctc_align_seqs.restype = C.c_int
    L.ccb_crf_sample_ws_bytes.argtypes = [i, i, i]; L.ccb_crf_sample_ws_bytes.restype = C.c_size_t
    L.ccb_crf_sample.argtypes = [vp, i, i, i, i, i, i, vp, i, C.c_uint64, i, vp, vp, vp, vp, vp, vp, vp, vp]
    L.ccb_crf_sample.restype = C.c_int
    L.ccb_ctc_beam_search_ws_bytes.argtypes = [i, i, i]; L.ccb_ctc_beam_search_ws_bytes.restype = C.c_size_t
    L.ccb_ctc_beam_search.argtypes = [vp, i, i, i, i, vp, i, i, i, vp, vp, vp, vp, vp, vp]
    L.ccb_ctc_beam_search.restype = C.c_int
    L.ccb_plan_ctc_shape.argtypes = [vp]; L.ccb_plan_ctc_shape.restype = C.c_int
    L.ccb_ngram_create.argtypes = [C.c_char_p, C.POINTER(C.c_char_p), i]; L.ccb_ngram_create.restype = vp
    L.ccb_ngram_destroy.argtypes = [vp]; L.ccb_ngram_destroy.restype = None
    L.ccb_ngram_info.argtypes = [vp, C.POINTER(C.c_long)]; L.ccb_ngram_info.restype = C.c_int
    L.ccb_ngram_copy.argtypes = [vp, i, vp, C.c_size_t]; L.ccb_ngram_copy.restype = C.c_int
    L.ccb_ctc_beam_search_lm.argtypes = [vp, i, i, i, i, vp, i, i, i, vp, vp, vp, vp, vp, vp, C.c_double, C.c_double, vp]
    L.ccb_ctc_beam_search_lm.restype = C.c_int
    L.ccb_wfst_create.argtypes = [C.c_char_p]; L.ccb_wfst_create.restype = vp
    L.ccb_wfst_destroy.argtypes = [vp]; L.ccb_wfst_destroy.restype = None
    L.ccb_wfst_info.argtypes = [vp, C.POINTER(C.c_long)]; L.ccb_wfst_info.restype = C.c_int
    L.ccb_wfst_copy.argtypes = [vp, i, vp, C.c_size_t]; L.ccb_wfst_copy.restype = C.c_int
    L.ccb_wfst_decode_ws_bytes.argtypes = [vp, i, i, i]; L.ccb_wfst_decode_ws_bytes.restype = C.c_size_t
    L.ccb_wfst_decode.argtypes = [vp, i, i, i, i, vp, vp, f, f, f, f, i, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.ccb_wfst_decode.restype = C.c_int
    L.ccb_rnnt_workspace_bytes.argtypes = [i, l]; L.ccb_rnnt_workspace_bytes.restype = C.c_size_t
    L.ccb_rnnt_forward.argtypes = [vp, i, i, i, i, l, i, i, i, vp, l, vp, vp, i, i, vp, vp, vp, vp]
    L.ccb_rnnt_forward.restype = C.c_int
    L.ccb_rnnt_backward.argtypes = [vp, i, i, i, l, i, vp, i, vp, vp, vp, vp]
    L.ccb_rnnt_backward.restype = C.c_int
    L.ccb_rnnt_simple_workspace_bytes.argtypes = [i, i, i]; L.ccb_rnnt_simple_workspace_bytes.restype = C.c_size_t
    L.ccb_rnnt_simple_forward.argtypes = [vp, vp, i, i, i, i, i, vp, vp, vp, i, i, vp, vp, vp]
    L.ccb_rnnt_simple_forward.restype = C.c_int
    L.ccb_rnnt_simple_backward.argtypes = [vp, vp, i, i, i, i, i, vp, i, vp, vp, vp, vp, vp]
    L.ccb_rnnt_simple_backward.restype = C.c_int
    for e in ("workspace_bytes", "forward", "backward", "simple_workspace_bytes", "simple_forward", "simple_backward"):
        # the CTC-T entries take the RNN-T entries' arguments
        getattr(L, f"ccb_ctct_{e}").argtypes = getattr(L, f"ccb_rnnt_{e}").argtypes
        getattr(L, f"ccb_ctct_{e}").restype = getattr(L, f"ccb_rnnt_{e}").restype
    L.ccb_rnnt_beam_ws_bytes.argtypes = [i, i, i]; L.ccb_rnnt_beam_ws_bytes.restype = C.c_size_t
    L.ccb_rnnt_beam_init.argtypes = [i, i, i, vp, vp, vp, vp, vp, vp]; L.ccb_rnnt_beam_init.restype = C.c_int
    L.ccb_rnnt_beam_step.argtypes = [vp, vp, i, i, i, i, i, i, i, vp, i, vp, vp, vp, vp, vp, vp]
    L.ccb_rnnt_beam_step.restype = C.c_int
    L.ccb_rnnt_beam_finish.argtypes = [i, i, i, i, vp, vp, vp, vp, vp, vp, vp]; L.ccb_rnnt_beam_finish.restype = C.c_int
    d = C.c_double
    L.ccb_rnnt_beam_step_fused.argtypes = L.ccb_rnnt_beam_step.argtypes[:-1] + [vp, i, d, d, vp, i, d, vp, vp]
    L.ccb_rnnt_beam_step_fused.restype = C.c_int
    L.ccb_ngram_slot_rows.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, vp]; L.ccb_ngram_slot_rows.restype = C.c_int
    L.ccb_lm_mix_slot_rows.argtypes = [i, vp, vp, vp, vp, i, vp, vp, vp, vp, i, i, i, vp, vp, vp, vp]
    L.ccb_lm_mix_slot_rows.restype = C.c_int
    L.ccb_ngram_score.argtypes = [vp, i, i, vp, l, i, vp, l, i, vp, i, vp, vp]; L.ccb_ngram_score.restype = C.c_int
    L.ccb_ctct_beam_ws_bytes.argtypes = [i, i, i]; L.ccb_ctct_beam_ws_bytes.restype = C.c_size_t
    L.ccb_ctct_beam_init.argtypes = [i, i, i, vp, vp, vp, vp, vp, vp]; L.ccb_ctct_beam_init.restype = C.c_int
    L.ccb_ctct_beam_step.argtypes = [vp, vp, i, i, i, i, i, i, i, vp, i, vp, vp, vp, vp, vp, vp]
    L.ccb_ctct_beam_step.restype = C.c_int
    L.ccb_gather_ws_bytes.argtypes = [i]; L.ccb_gather_ws_bytes.restype = C.c_size_t
    L.ccb_gather_sum.argtypes = [vp, vp, i, i, l, i, vp, vp, vp, vp, vp]; L.ccb_gather_sum.restype = C.c_int
    L.ccb_gather_sum_backward.argtypes = [vp, i, i, l, l, i, vp, vp, vp, vp, vp, vp]
    L.ccb_gather_sum_backward.restype = C.c_int
    L.ccb_launch_count.argtypes = []; L.ccb_launch_count.restype = C.c_long
    L.ccb_debug_timeline.argtypes = [vp, C.c_int, C.c_int]; L.ccb_debug_timeline.restype = None
    L.ccb_plan_create.argtypes = [C.c_char_p, C.c_int, C.c_int]; L.ccb_plan_create.restype = vp
    L.ccb_plan_destroy.argtypes = [vp]; L.ccb_plan_destroy.restype = None
    L.ccb_plan_info.argtypes = [vp, C.POINTER(C.c_long)]; L.ccb_plan_info.restype = C.c_int
    L.ccb_plan_copy.argtypes = [vp, C.c_int, vp, C.c_size_t]; L.ccb_plan_copy.restype = C.c_int
    L.ccb_plan_launch.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_long)]
    L.ccb_plan_launch.restype = C.c_int
    L.ccb_plan_launch_own.argtypes = L.ccb_plan_launch.argtypes
    L.ccb_plan_launch_own.restype = C.c_int
    _lib = L
    return L


def last_error() -> str:
    return lib().ccb_last_error().decode("utf-8", "replace")
