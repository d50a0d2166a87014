"""ctypes binding of include/w2l_b200.h for the Python harness (tests, bench, smoke).

Every function takes CUDA torch tensors, checks dtype/contiguity, and passes raw device
pointers and the current CUDA stream to the C ABI.  Workspaces are torch byte tensors owned
by the caller side (cached per size here), exactly as the C ABI demands.
"""
from __future__ import annotations

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libw2l_b200.so")

SCALE_MODES = {"none": 0, "input_sz": 1, "input_sz_sqrt": 2, "target_sz": 3, "target_sz_sqrt": 4}
TERM_FCC, TERM_FAC, TERM_ASG = 1, 2, 3

# every entry point include/w2l_b200.h declares (tests check the library exports all of them)
EXPORTS = [
    "w2l_version", "w2l_last_error", "w2l_launch_count", "w2l_reset_launch_count", "w2l_get_seed", "w2l_set_seed", "w2l_set_profile_events", "w2l_set_profile_event_list", "w2l_profile_events_used", "w2l_trace_begin", "w2l_trace_end", "w2l_trace_list",
    "w2l_asg_workspace_size", "w2l_asg_forward_backward",
    "w2l_asg64_workspace_size", "w2l_asg64_forward_backward",
    "w2l_fcc_viterbi_workspace_size", "w2l_fcc_viterbi",
    "w2l_fcc_viterbi64_workspace_size", "w2l_fcc_viterbi64",
    "w2l_fac_viterbi_workspace_size", "w2l_fac_viterbi",
    "w2l_ctc_workspace_size", "w2l_ctc_forward_backward", "w2l_argmax_path", "w2l_linseg_target",
    "w2l_ctc_viterbi_workspace_size", "w2l_ctc_viterbi_target",
    "w2l_set_precision", "w2l_get_precision", "w2l_gemm", "w2l_cast_bf16", "w2l_cast_bf16_rows", "w2l_cast_fp16", "w2l_cast_fp16_rows", "w2l_split_tf32", "w2l_sgd_step_ex", "w2l_finite_guard",
    "w2l_mask_bands", "w2l_trainer_set_precision", "w2l_trainer_set_grad_stream", "w2l_trainer_set_grad_stream_delay", "w2l_delay", "w2l_trainer_status", "w2l_trainer_save", "w2l_trainer_load", "w2l_trainer_export_streaming",
    "w2l_trainer_set_schedule", "w2l_trainer_set_position", "w2l_trainer_position", "w2l_trainer_set_lr", "w2l_trainer_lr",
    "w2l_trainer_set_amp", "w2l_trainer_amp_state",
    "w2l_text_create", "w2l_text_destroy", "w2l_text_num_classes", "w2l_text_encode", "w2l_text_prediction2ltr", "w2l_text_target2ltr",
    "w2l_text_ltr2wrd", "w2l_text_align_words", "w2l_edit_distance",
    "w2l_gemm_set_variant", "w2l_gemm_set_tile", "w2l_gemm_tf32", "w2l_gemm_tf32_ex", "w2l_gemm_tf32_view", "w2l_conv_time_workspace_size", "w2l_conv_time_fwd", "w2l_conv_time_dgrad",
    "w2l_conv_time_wgrad", "w2l_layernorm_fwd", "w2l_layernorm_rows_fwd", "w2l_layernorm_bwd", "w2l_colsum_accumulate", "w2l_sq_norm_accumulate",
    "w2l_sgd_step", "w2l_weightnorm_fwd", "w2l_weightnorm_bwd", "w2l_conv1d_arrange", "w2l_conv1d_arrange_ex", "w2l_conv1d_unarrange_grad",
    "w2l_glu_fwd", "w2l_glu_bwd", "w2l_prelu_fwd", "w2l_prelu_bwd", "w2l_transpose_input", "w2l_axpy", "w2l_fill", "w2l_act_fwd", "w2l_mask_mul",
    "w2l_trainer_create", "w2l_trainer_destroy", "w2l_trainer_step", "w2l_trainer_forward", "w2l_trainer_num_params",
    "w2l_trainer_param_layout", "w2l_trainer_get_flat", "w2l_trainer_set_flat", "w2l_trainer_sync_parameters",
    "w2l_trainer_describe", "w2l_nccl_unique_id", "w2l_init_distributed", "w2l_trainer_align", "w2l_trainer_time_stride",
    "w2l_mfsc_num_frames", "w2l_mfsc_workspace_size", "w2l_mfsc",
    "w2l_stream_create", "w2l_stream_destroy", "w2l_stream_state_bytes", "w2l_stream_max_frames_out", "w2l_stream_start",
    "w2l_stream_run", "w2l_stream_plan",
    "w2l_mfsc_stream_create", "w2l_mfsc_stream_destroy", "w2l_mfsc_stream_state_bytes", "w2l_mfsc_stream_max_frames_out",
    "w2l_mfsc_stream_start", "w2l_mfsc_stream_run",
    "w2l_seq2seq_check", "w2l_seq2seq_embed_fwd", "w2l_seq2seq_embed_bwd", "w2l_seq2seq_gru_stash_floats", "w2l_seq2seq_gru_fwd",
    "w2l_seq2seq_gru_bwd", "w2l_seq2seq_attn_fwd", "w2l_seq2seq_attn_bwd", "w2l_seq2seq_loss", "w2l_seq2seq_scale_rows",
    "w2l_seq2seq_decode_init", "w2l_seq2seq_decode_step",
    "w2l_seq2seq_beam_workspace_size", "w2l_seq2seq_beam_init", "w2l_seq2seq_beam_step", "w2l_seq2seq_beam_finish",
    "w2l_trainer_create_seq2seq", "w2l_trainer_output_width", "w2l_trainer_seq2seq_config", "w2l_trainer_clear_window",
    "w2l_trainer_seq2seq_seed", "w2l_trainer_decode", "w2l_trainer_beam_search",
    "w2l_seq2seq_sizes", "w2l_seq2seq_attn_fwd_sized", "w2l_seq2seq_attn_bwd_sized", "w2l_trainer_step_sized", "w2l_trainer_decode_sized",
    "w2l_trainer_beam_search_sized",
    "w2l_soft_label_loss", "w2l_ema_update", "w2l_trainer_set_ema", "w2l_trainer_ema", "w2l_trainer_forward_teacher",
    "w2l_trainer_viterbi_path", "w2l_trainer_step_soft",
    "w2l_text_device_create", "w2l_text_device_destroy", "w2l_text_edit_workspace_size", "w2l_text_edit_counts", "w2l_trainer_evaluate",
]


class W2LError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"w2l error {code}: {msg}")
        self.code = code


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / PyTorch fallback for the hot path)")
    lib = ctypes.CDLL(LIB_PATH)
    vp, i, sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t
    lib.w2l_last_error.restype = ctypes.c_char_p
    lib.w2l_launch_count.restype = ctypes.c_longlong
    lib.w2l_get_seed.restype = ctypes.c_ulonglong
    lib.w2l_set_seed.argtypes = [ctypes.c_ulonglong]
    lib.w2l_set_profile_events.argtypes = [vp, vp]
    lib.w2l_set_profile_event_list.argtypes = [i, vp, vp, i]
    lib.w2l_trace_begin.argtypes = [vp, i]
    lib.w2l_trace_end.restype = ctypes.c_longlong
    lib.w2l_trace_end.argtypes = [ctypes.c_char_p, ctypes.c_longlong]
    lib.w2l_trace_list.restype = ctypes.c_longlong
    lib.w2l_trace_list.argtypes = [ctypes.c_char_p, ctypes.c_longlong]
    lib.w2l_asg_workspace_size.restype = sz
    lib.w2l_asg_workspace_size.argtypes = [i, i, i, i]
    lib.w2l_asg_forward_backward.argtypes = [vp, i, i, i, i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, sz]
    lib.w2l_fcc_viterbi_workspace_size.restype = sz
    lib.w2l_fcc_viterbi_workspace_size.argtypes = [i, i, i]
    lib.w2l_fcc_viterbi.argtypes = [vp, i, i, i, vp, vp, vp, vp, sz]
    lib.w2l_asg64_workspace_size.restype = sz
    lib.w2l_asg64_workspace_size.argtypes = [i, i, i, i]
    lib.w2l_asg64_forward_backward.argtypes = [vp, i, i, i, i, i, i, vp, vp, vp, vp, vp, vp, vp, vp, sz]
    lib.w2l_fcc_viterbi64_workspace_size.restype = sz
    lib.w2l_fcc_viterbi64_workspace_size.argtypes = [i, i, i]
    lib.w2l_fcc_viterbi64.argtypes = [vp, i, i, i, vp, vp, vp, vp, sz]
    lib.w2l_fac_viterbi_workspace_size.restype = sz
    lib.w2l_fac_viterbi_workspace_size.argtypes = [i, i, i, i]
    lib.w2l_fac_viterbi.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, vp, vp, sz]
    lib.w2l_ctc_workspace_size.restype = sz
    lib.w2l_ctc_workspace_size.argtypes = [i, i, i, i]
    lib.w2l_ctc_forward_backward.argtypes = [vp, i, i, i, i, i, vp, vp, vp, vp, vp, vp, sz]
    lib.w2l_argmax_path.argtypes = [vp, i, i, i, vp, vp]
    lib.w2l_linseg_target.argtypes = [vp, i, i, i, vp, vp]
    lib.w2l_ctc_viterbi_workspace_size.restype = sz
    lib.w2l_ctc_viterbi_workspace_size.argtypes = [i, i, i, i]
    lib.w2l_ctc_viterbi_target.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, vp, sz]
    lib.w2l_gemm_tf32.argtypes = [vp, i, i, i, i, i, vp, i, vp, i, vp, i, vp, i]
    f32, u64, ll = ctypes.c_float, ctypes.c_ulonglong, ctypes.c_longlong
    ll = ctypes.c_longlong
    lib.w2l_weightnorm_fwd.argtypes = [vp, i, i, vp, vp, vp, vp]
    lib.w2l_weightnorm_bwd.argtypes = [vp, i, i, vp, vp, vp, vp, vp, vp]
    lib.w2l_conv1d_arrange.argtypes = [vp, i, i, i, i, i, i, vp, vp, vp, vp, vp]
    lib.w2l_conv1d_unarrange_grad.argtypes = [vp, i, i, i, i, i, i, vp, vp, ll, vp, vp]
    lib.w2l_glu_fwd.argtypes = [vp, ll, i, vp, vp, f32, u64]
    lib.w2l_glu_bwd.argtypes = [vp, ll, i, vp, vp, vp, f32, u64]
    lib.w2l_prelu_fwd.argtypes = [vp, ll, vp, vp, vp, f32, u64]
    lib.w2l_prelu_bwd.argtypes = [vp, ll, vp, vp, vp, vp, vp, f32, u64]
    lib.w2l_act_fwd.argtypes = [vp, ll, vp, i, f32, u64, vp]
    lib.w2l_mask_mul.argtypes = [vp, ll, vp, vp, i, f32, vp]
    lib.w2l_gemm_tf32_view.argtypes = [vp, i, i, i, i, i, vp, i, vp, i, vp, i, vp, i, i]
    lib.w2l_gemm_tf32_ex.argtypes = [vp, i, i, i, i, i, vp, i, vp, i, vp, i, vp, i, i, vp, i, i, f32, f32, u64]
    lib.w2l_conv_time_workspace_size.restype = sz
    lib.w2l_conv_time_workspace_size.argtypes = [i, i, i, i, i]
    lib.w2l_conv_time_fwd.argtypes = [vp, i, i, i, i, i, i, i, i, i, vp, vp, vp, vp, vp, i, f32, u64, vp, sz]
    lib.w2l_conv_time_dgrad.argtypes = [vp, i, i, i, i, i, i, i, i, i, vp, vp, vp, vp, vp, sz]
    lib.w2l_conv_time_wgrad.argtypes = [vp, i, i, i, i, i, i, i, i, i, vp, vp, vp, vp, vp, sz]
    lib.w2l_layernorm_fwd.argtypes = [vp, i, ll, f32, vp, vp, vp, vp, vp, vp, vp]
    lib.w2l_layernorm_rows_fwd.argtypes = [vp, ll, i, f32, vp, vp, vp, vp, vp, vp]
    lib.w2l_layernorm_bwd.argtypes = [vp, i, ll, vp, vp, vp, vp, vp, vp, vp, i, f32, vp, vp, vp]
    lib.w2l_colsum_accumulate.argtypes = [vp, i, i, vp, i, vp]
    lib.w2l_sq_norm_accumulate.argtypes = [vp, ll, vp, vp]
    lib.w2l_sgd_step.argtypes = [vp, ll, vp, vp, vp, f32, f32, f32, f32, f32, vp]
    lib.w2l_set_precision.argtypes = [i]
    lib.w2l_gemm.argtypes = [vp, i, i, i, i, i, i, vp, i, vp, i, vp, i, i, vp, i, i, vp, i, i, i, f32, f32, u64, i]
    lib.w2l_cast_bf16.argtypes = [vp, ll, vp, vp]
    lib.w2l_cast_bf16_rows.argtypes = [vp, ll, i, i, i, vp, vp]
    lib.w2l_cast_fp16.argtypes = [vp, ll, vp, vp]
    lib.w2l_cast_fp16_rows.argtypes = [vp, ll, i, i, i, vp, vp]
    lib.w2l_split_tf32.argtypes = [vp, i, i, i, i, i, vp, vp]
    lib.w2l_sgd_step_ex.argtypes = [vp, ll, vp, vp, vp, f32, f32, f32, f32, f32, vp, i, vp]
    lib.w2l_finite_guard.argtypes = [vp, i, vp, vp, vp]
    lib.w2l_mask_bands.argtypes = [vp, i, i, i, i, vp, vp, i, vp, vp, i, vp, vp, f32]
    lib.w2l_trainer_set_precision.argtypes = [vp, i]
    lib.w2l_trainer_set_schedule.argtypes = [vp, ll, ctypes.c_double, ll, i, ll, ll, ll]
    lib.w2l_trainer_set_position.argtypes = [vp, ll, ll]
    lib.w2l_trainer_position.argtypes = [vp, vp, vp]
    lib.w2l_trainer_set_lr.argtypes = [vp, ctypes.c_float, ctypes.c_float]
    lib.w2l_trainer_lr.argtypes = [vp, vp, vp]
    lib.w2l_trainer_set_amp.argtypes = [vp, i, ctypes.c_double, i, ctypes.c_double, ctypes.c_double]
    lib.w2l_trainer_amp_state.argtypes = [vp, vp, vp, vp, vp]
    lib.w2l_trainer_set_grad_stream.argtypes = [vp, i]
    lib.w2l_trainer_set_grad_stream_delay.argtypes = [vp, i]
    lib.w2l_delay.argtypes = [vp, i]
    lib.w2l_trainer_status.argtypes = [vp, vp, vp]
    cp = ctypes.c_char_p
    lib.w2l_trainer_save.argtypes = [vp, vp, cp]
    lib.w2l_trainer_load.restype = vp
    lib.w2l_trainer_load.argtypes = [vp, cp]
    lib.w2l_trainer_export_streaming.argtypes = [vp, vp, cp, cp]
    lib.w2l_text_create.restype = vp
    lib.w2l_text_create.argtypes = [cp, cp, cp, i, cp, i, cp]
    lib.w2l_text_destroy.argtypes = [vp]
    lib.w2l_text_destroy.restype = None
    lib.w2l_text_num_classes.argtypes = [vp]
    for fn in (lib.w2l_text_encode, lib.w2l_text_prediction2ltr, lib.w2l_text_target2ltr, lib.w2l_text_ltr2wrd):
        fn.restype = ll
    lib.w2l_text_encode.argtypes = [vp, cp, vp, ll]
    lib.w2l_text_prediction2ltr.argtypes = [vp, vp, i, vp, ll]
    lib.w2l_text_target2ltr.argtypes = [vp, vp, i, vp, ll]
    lib.w2l_text_ltr2wrd.argtypes = [vp, cp, vp, ll]
    lib.w2l_text_align_words.restype = ll
    lib.w2l_text_align_words.argtypes = [vp, vp, i, vp, i, ctypes.c_double, cp, vp, ll]
    lib.w2l_edit_distance.argtypes = [cp, cp, vp]
    lib.w2l_text_device_create.restype = vp
    lib.w2l_text_device_create.argtypes = [vp, vp]
    lib.w2l_text_device_destroy.argtypes = [vp]
    lib.w2l_text_device_destroy.restype = None
    lib.w2l_text_edit_workspace_size.restype = sz
    lib.w2l_text_edit_workspace_size.argtypes = [vp, i, i, i]
    lib.w2l_text_edit_counts.argtypes = [vp, vp, i, i, vp, vp, i, vp, vp, vp, sz]
    lib.w2l_trainer_evaluate.argtypes = [vp, vp, vp, i, i, vp, i, vp, vp, vp, vp, vp]
    lib.w2l_trainer_create.restype = vp
    lib.w2l_trainer_create.argtypes = [vp, ctypes.c_char_p, i, i, ctypes.c_char_p, i, f32, f32, f32, f32, f32]
    lib.w2l_trainer_create_seq2seq.restype = vp
    lib.w2l_trainer_create_seq2seq.argtypes = [vp, ctypes.c_char_p, i, i, i, i, i, i, i, i, f32, f32, i, f32, i, f32, f32, f32, f32]
    lib.w2l_trainer_output_width.argtypes = [vp, vp]
    lib.w2l_trainer_seq2seq_config.argtypes = [vp, vp]
    lib.w2l_trainer_clear_window.argtypes = [vp]
    lib.w2l_trainer_seq2seq_seed.argtypes = [vp, vp]
    lib.w2l_trainer_decode.argtypes = [vp, vp, i, i, vp, vp, vp, ll]
    lib.w2l_trainer_beam_search.argtypes = [vp, vp, i, i, vp, i, i, vp, vp, vp, vp, ll]
    lib.w2l_seq2seq_check.argtypes = [i, i]
    lib.w2l_seq2seq_embed_fwd.argtypes = [vp, i, i, i, i, vp, vp, vp, f32, u64, vp, vp, vp]
    lib.w2l_seq2seq_embed_bwd.argtypes = [vp, i, i, i, i, vp, vp, vp, vp]
    lib.w2l_seq2seq_gru_stash_floats.restype = sz
    lib.w2l_seq2seq_gru_stash_floats.argtypes = [i, i, i]
    lib.w2l_seq2seq_gru_fwd.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, vp]
    lib.w2l_seq2seq_gru_bwd.argtypes = [vp, i, i, i, vp, vp, vp, vp, vp, vp]
    lib.w2l_seq2seq_attn_fwd.argtypes = [vp, i, i, i, i, vp, vp, i, f32, vp, vp]
    lib.w2l_seq2seq_attn_bwd.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, vp, vp, vp]
    lib.w2l_seq2seq_sizes.argtypes = [vp, i, i, i, vp, i, vp, vp, vp, vp]
    lib.w2l_seq2seq_attn_fwd_sized.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, i, f32, vp, vp]
    lib.w2l_seq2seq_attn_bwd_sized.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.w2l_trainer_step_sized.argtypes = [vp, vp, i, i, vp, i, vp, vp, vp, vp, i, f32]
    lib.w2l_trainer_decode_sized.argtypes = [vp, vp, i, i, vp, vp, vp, vp, ll]
    lib.w2l_trainer_beam_search_sized.argtypes = [vp, vp, i, i, vp, vp, i, i, vp, vp, vp, vp, ll]
    lib.w2l_seq2seq_loss.argtypes = [vp, i, i, i, i, vp, vp, f32, vp, i, vp, vp, vp]
    lib.w2l_seq2seq_scale_rows.argtypes = [vp, i, i, i, vp, f32, vp]
    lib.w2l_seq2seq_decode_init.argtypes = [vp, i, i, i, i, vp, vp, vp, vp, vp]
    lib.w2l_seq2seq_decode_step.argtypes = [vp, i, i, i, i, i, vp, vp, vp, vp, i, vp, vp]
    lib.w2l_seq2seq_beam_workspace_size.restype = sz
    lib.w2l_seq2seq_beam_workspace_size.argtypes = [i, i, i]
    lib.w2l_seq2seq_beam_init.argtypes = [vp, i, i, i, i, vp, vp, vp, sz]
    lib.w2l_seq2seq_beam_step.argtypes = [vp, i, i, i, i, i, i, i, i, vp, vp, vp, vp, vp, vp, sz]
    lib.w2l_seq2seq_beam_finish.argtypes = [vp, i, i, i, i, i, vp, sz, vp, vp, vp, vp]
    lib.w2l_trainer_destroy.argtypes = [vp]
    lib.w2l_trainer_destroy.restype = None
    lib.w2l_trainer_step.argtypes = [vp, vp, i, i, vp, i, vp, vp, i, f32]
    lib.w2l_trainer_forward.argtypes = [vp, vp, i, i, vp, vp, ll, vp]
    lib.w2l_soft_label_loss.argtypes = [vp, ll, i, vp, vp, f32, vp, vp, vp]
    lib.w2l_ema_update.argtypes = [vp, ll, vp, vp, ctypes.c_double]
    lib.w2l_trainer_set_ema.argtypes = [vp, vp, i, ctypes.c_double]
    lib.w2l_trainer_ema.argtypes = [vp, vp, vp]
    lib.w2l_trainer_forward_teacher.argtypes = [vp, vp, i, i, vp, i, vp, ll, vp]
    lib.w2l_trainer_viterbi_path.argtypes = [vp, vp, i, i, vp, vp, i, vp, ll, vp]
    lib.w2l_trainer_step_soft.argtypes = [vp, vp, i, i, vp, vp, i, f32, vp, f32]
    lib.w2l_trainer_align.argtypes = [vp, vp, i, i, vp, i, vp, vp, vp, ll, vp]
    lib.w2l_trainer_time_stride.argtypes = [vp]
    lib.w2l_trainer_num_params.restype = ll
    lib.w2l_trainer_num_params.argtypes = [vp, i]
    lib.w2l_trainer_param_layout.argtypes = [vp, i, i, vp, vp]
    lib.w2l_trainer_get_flat.argtypes = [vp, vp, i, i, vp]
    lib.w2l_trainer_set_flat.argtypes = [vp, vp, i, vp]
    lib.w2l_trainer_sync_parameters.argtypes = [vp, vp]
    lib.w2l_trainer_describe.restype = ctypes.c_char_p
    lib.w2l_trainer_describe.argtypes = [vp]
    lib.w2l_nccl_unique_id.argtypes = [vp]
    lib.w2l_init_distributed.argtypes = [i, i, vp]
    lib.w2l_mfsc_num_frames.argtypes = [i, i, i, i]
    lib.w2l_mfsc_workspace_size.restype = sz
    lib.w2l_mfsc_workspace_size.argtypes = [i, i, i, i, i, i]
    lib.w2l_mfsc.argtypes = [vp, i, i, vp, vp, i, i, i, i, i, vp, i, vp, sz]
    lib.w2l_stream_create.restype = vp
    lib.w2l_stream_create.argtypes = [vp, vp, i, i]
    lib.w2l_stream_destroy.argtypes = [vp]
    lib.w2l_stream_destroy.restype = None
    lib.w2l_stream_state_bytes.restype = ctypes.c_longlong
    lib.w2l_stream_state_bytes.argtypes = [vp]
    lib.w2l_stream_max_frames_out.argtypes = [vp]
    lib.w2l_stream_start.argtypes = [vp, vp, i, vp]
    lib.w2l_stream_run.argtypes = [vp, vp, i, vp, vp, vp, i, i, vp, ctypes.c_longlong, vp]
    lib.w2l_stream_plan.argtypes = [ctypes.c_char_p, i, i, i, vp, i, i, vp, vp, vp, vp]
    lib.w2l_mfsc_stream_create.restype = vp
    lib.w2l_mfsc_stream_create.argtypes = [vp, i, i, i, i, i, i, i]
    lib.w2l_mfsc_stream_destroy.argtypes = [vp]
    lib.w2l_mfsc_stream_destroy.restype = None
    lib.w2l_mfsc_stream_state_bytes.restype = ctypes.c_longlong
    lib.w2l_mfsc_stream_state_bytes.argtypes = [vp]
    lib.w2l_mfsc_stream_max_frames_out.argtypes = [vp]
    lib.w2l_mfsc_stream_start.argtypes = [vp, vp, i, vp]
    lib.w2l_mfsc_stream_run.argtypes = [vp, vp, i, vp, vp, vp, i, i, vp, ctypes.c_longlong, vp]
    return lib


lib = _load()


def _check(rc: int) -> None:
    if rc != 0:
        raise W2LError(rc, lib.w2l_last_error().decode())


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _req(t, dtype, name):
    if t is None:
        return None
    if not t.is_cuda or t.dtype != dtype or not t.is_contiguous():
        raise TypeError(f"{name}: expected a contiguous CUDA tensor of {dtype}")
    return t


_ws_cache: dict = {}


def workspace(nbytes: int, device) -> torch.Tensor:
    key = (str(device), "ws")
    t = _ws_cache.get(key)
    if t is None or t.numel() < nbytes:
        t = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=device)
        _ws_cache[key] = t
    return t


def _mode(m) -> int:
    return SCALE_MODES[m] if isinstance(m, str) else int(m)


def launch_count() -> int:
    return int(lib.w2l_launch_count())


def reset_launch_count() -> None:
    lib.w2l_reset_launch_count()


def set_profile_events(start=None, stop=None) -> None:
    """torch.cuda.Event(enable_timing=True) pair recorded around each call's dominant kernel."""
    if start is None:
        lib.w2l_set_profile_events(None, None)
    else:
        start.record()  # make sure the lazily created handles exist
        stop.record()
        lib.w2l_set_profile_events(ctypes.c_void_p(start.cuda_event), ctypes.c_void_p(stop.cuda_event))


def asg_forward_backward(emis, target, trans, scale_mode="none", dloss=None, terms=TERM_ASG, need_grad=True,
                         out=None, ws=None):
    """Fused ASG (FCC - FAC) forward+backward.  emis [B,T,N] f32, target [B,L] i32 (-1 padded),
    trans [N,N] f32.  Returns (loss[B], d_emis[B,T,N] | None, d_trans[N,N] | None).  N <= 32."""
    return _asg(lib.w2l_asg_workspace_size, lib.w2l_asg_forward_backward, emis, target, trans, scale_mode, dloss,
                terms, need_grad, out, ws)


def asg64_forward_backward(emis, target, trans, scale_mode="none", dloss=None, terms=TERM_ASG, need_grad=True,
                           out=None, ws=None):
    """asg_forward_backward for 1 <= N <= 64 (w2l_asg64_forward_backward)."""
    return _asg(lib.w2l_asg64_workspace_size, lib.w2l_asg64_forward_backward, emis, target, trans, scale_mode, dloss,
                terms, need_grad, out, ws)


def _asg(ws_size, call, emis, target, trans, scale_mode, dloss, terms, need_grad, out, ws):
    emis = _req(emis, torch.float32, "emis")
    trans = _req(trans, torch.float32, "trans")
    target = _req(target, torch.int32, "target")
    dloss = _req(dloss, torch.float32, "dloss")
    B, T, N = emis.shape
    L = 0 if target is None else target.shape[1]
    if out is None:
        loss = torch.empty(B, dtype=torch.float32, device=emis.device)
        d_emis = torch.empty_like(emis) if need_grad else None
        d_trans = torch.empty_like(trans) if need_grad else None
    else:
        loss, d_emis, d_trans = out
    need = ws_size(B, T, N, L)
    if ws is None:
        ws = workspace(need, emis.device)
    _check(call(_stream(), terms, B, T, N, L, _mode(scale_mode), _ptr(emis), _ptr(target),
                _ptr(trans), _ptr(dloss), _ptr(loss), _ptr(d_emis), _ptr(d_trans),
                _ptr(ws), ws.numel()))
    return loss, d_emis, d_trans


def prelu_fwd(x, a, dropout_p=0.0, seed=0):
    """PReLU with one parameter and the fused dropout (the `PR` opcode's kernel): x CUDA float32, a CUDA float32 [1]."""
    x = _req(x, torch.float32, "x")
    a = _req(a, torch.float32, "a")
    y = torch.empty_like(x)
    _check(lib.w2l_prelu_fwd(_stream(), x.numel(), _ptr(x), _ptr(a), _ptr(y), float(dropout_p), int(seed)))
    return y


def prelu_bwd(x, dy, a, dropout_p=0.0, seed=0):
    """(dx, da [1]) of prelu_fwd for the upstream gradient dy; the dropout mask is regenerated from seed."""
    x = _req(x, torch.float32, "x")
    dy = _req(dy, torch.float32, "dy")
    a = _req(a, torch.float32, "a")
    dx = torch.empty_like(x)
    da = torch.empty(1, dtype=torch.float32, device=x.device)
    _check(lib.w2l_prelu_bwd(_stream(), x.numel(), _ptr(x), _ptr(dy), _ptr(a), _ptr(dx), _ptr(da), float(dropout_p), int(seed)))
    return dx, da


def fcc_viterbi(emis, trans):
    """Max-plus FCC Viterbi path [B,T] i32, N <= 32."""
    return _fcc_viterbi(lib.w2l_fcc_viterbi_workspace_size, lib.w2l_fcc_viterbi, emis, trans)


def fcc_viterbi64(emis, trans):
    """fcc_viterbi for 1 <= N <= 64 (w2l_fcc_viterbi64), bit-exact like it."""
    return _fcc_viterbi(lib.w2l_fcc_viterbi64_workspace_size, lib.w2l_fcc_viterbi64, emis, trans)


def _fcc_viterbi(ws_size, call, emis, trans):
    emis = _req(emis, torch.float32, "emis")
    trans = _req(trans, torch.float32, "trans")
    B, T, N = emis.shape
    path = torch.empty((B, T), dtype=torch.int32, device=emis.device)
    ws = workspace(ws_size(B, T, N), emis.device)
    _check(call(_stream(), B, T, N, _ptr(emis), _ptr(trans), _ptr(path), _ptr(ws), ws.numel()))
    return path


def fac_viterbi(emis, target, trans, return_index=False):
    emis = _req(emis, torch.float32, "emis")
    trans = _req(trans, torch.float32, "trans")
    target = _req(target, torch.int32, "target")
    B, T, N = emis.shape
    L = target.shape[1]
    path = torch.empty((B, T), dtype=torch.int32, device=emis.device)
    idx = torch.empty((B, T), dtype=torch.int32, device=emis.device) if return_index else None
    ws = workspace(lib.w2l_fac_viterbi_workspace_size(B, T, N, L), emis.device)
    _check(lib.w2l_fac_viterbi(_stream(), B, T, N, L, _ptr(emis), _ptr(target), _ptr(trans), _ptr(path), _ptr(idx),
                               _ptr(ws), ws.numel()))
    return (path, idx) if return_index else path


def ctc_forward_backward(emis, target, scale_mode="none", dloss=None, need_grad=True, out=None, ws=None):
    """CTC on raw activations (blank = N-1).  Returns (loss[B], d_emis | None)."""
    emis = _req(emis, torch.float32, "emis")
    target = _req(target, torch.int32, "target")
    dloss = _req(dloss, torch.float32, "dloss")
    B, T, N = emis.shape
    L = 0 if target is None else target.shape[1]
    if out is None:
        loss = torch.empty(B, dtype=torch.float32, device=emis.device)
        d_emis = torch.empty_like(emis) if need_grad else None
    else:
        loss, d_emis = out
    need = lib.w2l_ctc_workspace_size(B, T, N, L)
    if ws is None:
        ws = workspace(need, emis.device)
    _check(lib.w2l_ctc_forward_backward(_stream(), B, T, N, L, _mode(scale_mode), _ptr(emis), _ptr(target),
                                        _ptr(dloss), _ptr(loss), _ptr(d_emis), _ptr(ws), ws.numel()))
    return loss, d_emis


def argmax_path(emis):
    emis = _req(emis, torch.float32, "emis")
    B, T, N = emis.shape
    path = torch.empty((B, T), dtype=torch.int32, device=emis.device)
    _check(lib.w2l_argmax_path(_stream(), B, T, N, _ptr(emis), _ptr(path)))
    return path


def ctc_viterbi_target(emis, target, return_state=False):
    """CTC forced alignment on raw activations (blank = N-1): path [B,T] int32 (label or blank per frame, -1 for a
    target that cannot be aligned) and, with return_state, the extended-target state per frame."""
    emis = _req(emis, torch.float32, "emis")
    target = _req(target, torch.int32, "target")
    B, T, N = emis.shape
    L = target.shape[1]
    path = torch.empty((B, T), dtype=torch.int32, device=emis.device)
    state = torch.empty((B, T), dtype=torch.int32, device=emis.device) if return_state else None
    ws = workspace(lib.w2l_ctc_viterbi_workspace_size(B, T, N, L), emis.device)
    _check(lib.w2l_ctc_viterbi_target(_stream(), B, T, N, L, _ptr(emis), _ptr(target), _ptr(path), _ptr(state), _ptr(ws),
                                      ws.numel()))
    return (path, state) if return_state else path


def linseg_target(target, T: int):
    target = _req(target, torch.int32, "target")
    B, L = target.shape
    out = torch.empty((B, int(T)), dtype=torch.int32, device=target.device)
    _check(lib.w2l_linseg_target(_stream(), B, int(T), L, _ptr(target), _ptr(out)))
    return out


class ProfileList:
    """n CUDA event pairs recorded around the dominant-kernel launches of `kind` (1 GEMM, 2 criterion chains)."""

    def __init__(self, kind: int, n: int):
        self.starts = [torch.cuda.Event(enable_timing=True) for _ in range(n)]
        self.stops = [torch.cuda.Event(enable_timing=True) for _ in range(n)]
        for e in self.starts + self.stops:
            e.record()
        self._a = (ctypes.c_void_p * n)(*[e.cuda_event for e in self.starts])
        self._b = (ctypes.c_void_p * n)(*[e.cuda_event for e in self.stops])
        self.kind, self.n = kind, n

    def arm(self):
        lib.w2l_set_profile_event_list(self.kind, self._a, self._b, self.n)

    def disarm(self) -> int:
        used = int(lib.w2l_profile_events_used())
        lib.w2l_set_profile_event_list(0, None, None, 0)
        return used

    def times_ms(self, used: int):
        return [self.starts[k].elapsed_time(self.stops[k]) for k in range(used)]


def trace_list() -> list:
    """every launch of the last trace() in order: [(kernel name, ms)]"""
    buf = ctypes.create_string_buffer(1 << 18)
    lib.w2l_trace_list(buf, len(buf))
    return [(ln.split("\t")[0], float(ln.split("\t")[1])) for ln in buf.value.decode().splitlines()]


PRECISIONS = {"tf32": 0, "f32": 1, "fp32": 1, "bf16": 2, "fp16": 3}
GEMM_KINDS = {"tf32": 0, "f32x3": 1, "bf16": 2, "f32x3_split_b": 3, "fp16": 4}


def set_precision(p) -> None:
    """tf32 (default) | f32 (fp32-accurate 3xTF32 GEMMs and mma.sync time convolutions) | bf16 (bf16 GEMM operands) |
    fp16 (fp16 GEMM operands)."""
    _check(lib.w2l_set_precision(PRECISIONS[p] if isinstance(p, str) else int(p)))


def get_precision() -> int:
    return int(lib.w2l_get_precision())


def gemm(A, B, kind="tf32", a_mn=False, b_mn=False, bias=None, act=0, out=None, out_bf16=False, accumulate=False, aux=None,
         aux_mode=0, aux_scale=1.0, dropout_p=0.0, seed=0, M=None, N=None, K=None, lda=None, ldb=None, allow_overlap=False):
    """General wgmma GEMM (w2l_gemm): A/B fp32 (kinds tf32, f32x3), bfloat16 (kind bf16) or float16 (kind fp16); C fp32 or
    16-bit (out_bf16: float16 for kind fp16, bfloat16 otherwise), aux likewise.
    Kind f32x3_split_b: B is the [2][N][ldb] planes of split_tf32 (K is taken from A)."""
    if M is None:
        M, K = (A.shape[1], A.shape[0]) if a_mn else A.shape
        N = B.shape[-2] if B.dim() == 3 else (B.shape[1] if b_mn else B.shape[0])
    lda = A.stride(0) if lda is None else lda
    ldb = B.stride(-2) if ldb is None else ldb
    kind_id = GEMM_KINDS[kind] if isinstance(kind, str) else int(kind)
    half = torch.float16 if kind_id == GEMM_KINDS["fp16"] else torch.bfloat16  # the kind's 16-bit C / aux type
    if out is None:
        out = torch.empty((M, N), dtype=half if out_bf16 else torch.float32, device=A.device)
    if out.dtype not in (torch.float32, half) or (aux is not None and aux.dtype not in (torch.float32, half)):
        raise TypeError(f"gemm: a 16-bit C or aux of kind {kind} is {half}")
    _check(lib.w2l_gemm(_stream(), kind_id, int(a_mn), int(b_mn), M, N, K, _ptr(A), lda, _ptr(B), ldb, _ptr(out),
                        out.stride(0), int(out.dtype == half), _ptr(bias), int(act), int(accumulate), _ptr(aux),
                        0 if aux is None else aux.stride(0), int(aux is not None and aux.dtype == half),
                        int(aux_mode), float(aux_scale), float(dropout_p), int(seed), int(allow_overlap)))
    return out


def cast_bf16(x):
    x = _req(x, torch.float32, "x")
    y = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _check(lib.w2l_cast_bf16(_stream(), x.numel(), _ptr(x), _ptr(y)))
    return y


def cast_fp16(x):
    x = _req(x, torch.float32, "x")
    y = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _check(lib.w2l_cast_fp16(_stream(), x.numel(), _ptr(x), _ptr(y)))
    return y


def cast_fp16_rows(x, cols_padded):
    """rows of a 2-D fp32 tensor (rows contiguous) -> [rows][cols_padded] float16, zero-padded columns"""
    x = _req(x, torch.float32, "x")
    if x.dim() != 2 or x.stride(1) != 1:
        raise TypeError("cast_fp16_rows: x must be 2-D with contiguous rows")
    y = torch.empty((x.shape[0], cols_padded), dtype=torch.float16, device=x.device)
    _check(lib.w2l_cast_fp16_rows(_stream(), x.shape[0], x.shape[1], x.stride(0), cols_padded, _ptr(x), _ptr(y)))
    return y


def split_tf32(x, transpose=False, cols_padded=None):
    """B planes of kind f32x3_split_b from a 2-D fp32 tensor x (rows contiguous): [2][rows][cols_padded] tf32 hi / lo,
    or with transpose those of x^T, [2][cols][cols_padded]; cols_padded defaults to the source row length rounded up
    to 4 (a TMA row)"""
    if x.dtype != torch.float32 or not x.is_cuda or x.dim() != 2 or x.stride(1) != 1:
        raise TypeError("split_tf32: x must be a 2-D CUDA float32 tensor with contiguous rows")
    rows, cols = x.shape
    k = rows if transpose else cols
    cols_padded = (k + 3) // 4 * 4 if cols_padded is None else cols_padded
    y = torch.empty((2, cols if transpose else rows, cols_padded), dtype=torch.float32, device=x.device)
    _check(lib.w2l_split_tf32(_stream(), int(transpose), rows, cols, x.stride(0), cols_padded, _ptr(x), _ptr(y)))
    return y


def gemm_set_variant(v: int = 1):
    """1: one CTA per SM walking the tiles (default); 0: one tile per CTA"""
    _check(lib.w2l_gemm_set_variant(int(v)))


def gemm_set_tile(bn: int = 0):
    _check(lib.w2l_gemm_set_tile(int(bn)))


def trace(fn, capacity: int = 4096) -> dict:
    """Run fn() (all work on the current stream) in trace mode; returns {kernel name: (launches, total ms)} measured
    with one CUDA event after every launch — the warm, in-situ share of each kernel (measurement only)."""
    _check(lib.w2l_trace_begin(_stream(), capacity))
    try:
        fn()
    finally:
        buf = ctypes.create_string_buffer(1 << 16)
        lib.w2l_trace_end(buf, len(buf))
    out = {}
    for line in buf.value.decode().splitlines():
        name, n, ms = line.split("\t")
        out[name] = (int(n), float(ms))
    return out


def gemm_tf32(A, B, bias=None, act=0, a_mn=False, b_mn=False, out=None):
    """C[m][n] = act(sum_k A(m,k) B(n,k) + bias[n]).  A: [M,K] (or [K,M] if a_mn), B: [N,K] (or [K,N] if b_mn)."""
    A = _req(A, torch.float32, "A")
    B = _req(B, torch.float32, "B")
    bias = _req(bias, torch.float32, "bias")
    M, K = (A.shape[1], A.shape[0]) if a_mn else A.shape
    N = B.shape[1] if b_mn else B.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=A.device)
    _check(lib.w2l_gemm_tf32(_stream(), int(a_mn), int(b_mn), M, N, K, _ptr(A), A.stride(0), _ptr(B), B.stride(0),
                             _ptr(out), out.stride(0), _ptr(bias), int(act)))
    return out


def gemm_tf32_ex(A, B, out, bias=None, act=0, a_mn=False, b_mn=False, accumulate=False, aux=None, aux_mode=0,
                 aux_scale=1.0, dropout_p=0.0, seed=0):
    M, K = (A.shape[1], A.shape[0]) if a_mn else A.shape
    N = B.shape[1] if b_mn else B.shape[0]
    _check(lib.w2l_gemm_tf32_ex(_stream(), int(a_mn), int(b_mn), M, N, K, _ptr(A), A.stride(0), _ptr(B), B.stride(0),
                                _ptr(out), out.stride(0), _ptr(bias), int(act), int(accumulate), _ptr(aux),
                                0 if aux is None else aux.stride(0), int(aux_mode), float(aux_scale), float(dropout_p),
                                int(seed)))
    return out


def gemm_tf32_view(A, lda, B, ldb, out, M, N, K, a_mn=False, b_mn=False, bias=None, act=0, accumulate=False):
    """GEMM on raw (possibly overlapping-row) operand views: A/B are any CUDA float tensors, lda/ldb explicit."""
    _check(lib.w2l_gemm_tf32_view(_stream(), int(a_mn), int(b_mn), M, N, K, _ptr(A), lda, _ptr(B), ldb, _ptr(out), out.stride(0),
                                  _ptr(bias), int(act), int(accumulate)))
    return out


def conv_time_ws(B, Tout, Cin, Cout, K, device):
    return workspace(lib.w2l_conv_time_workspace_size(B, Tout, Cin, Cout, K), device)


def conv_time_fwd(x, wt, bias, Tout, stride, pad_left, act=0, dropout_p=0.0, seed=0, add=None):
    """x [B,T,Cin,W], wt [Cout,Cin,K] -> y [B,Tout,Cout,W]"""
    B, T, Cin, W = x.shape
    Cout, _, K = wt.shape
    y = torch.empty((B, Tout, Cout, W), dtype=torch.float32, device=x.device)
    ws = conv_time_ws(B, Tout, Cin, Cout, K, x.device)
    _check(lib.w2l_conv_time_fwd(_stream(), B, T, Tout, W, Cin, Cout, K, stride, pad_left, _ptr(x), _ptr(wt), _ptr(bias),
                                 _ptr(add), _ptr(y), act, float(dropout_p), int(seed), _ptr(ws), ws.numel()))
    return y


def conv_time_dgrad(dy, wt, T, stride, pad_left, add=None, out=None):
    """dx = conv^T(dy) (+ add); out may be the same tensor as add (in-place accumulation)."""
    B, Tout, Cout, W = dy.shape
    _, Cin, K = wt.shape
    dx = out if out is not None else torch.empty((B, T, Cin, W), dtype=torch.float32, device=dy.device)
    ws = conv_time_ws(B, Tout, Cin, Cout, K, dy.device)
    _check(lib.w2l_conv_time_dgrad(_stream(), B, T, Tout, W, Cin, Cout, K, stride, pad_left, _ptr(dy), _ptr(wt), _ptr(add),
                                   _ptr(dx), _ptr(ws), ws.numel()))
    return dx


def conv_time_wgrad(x, dy, K, stride, pad_left, dwt=None, dbias=None):
    B, T, Cin, W = x.shape
    _, Tout, Cout, _ = dy.shape
    if dwt is None:
        dwt = torch.zeros((Cout, Cin, K), dtype=torch.float32, device=x.device)
        dbias = torch.zeros(Cout, dtype=torch.float32, device=x.device)
    ws = conv_time_ws(B, Tout, Cin, Cout, K, x.device)
    _check(lib.w2l_conv_time_wgrad(_stream(), B, T, Tout, W, Cin, Cout, K, stride, pad_left, _ptr(x), _ptr(dy), _ptr(dwt),
                                   _ptr(dbias), _ptr(ws), ws.numel()))
    return dwt, dbias


def layernorm_fwd(a, r, gain, bias, eps=1e-5):
    B = a.shape[0]
    R = a[0].numel()
    y = torch.empty_like(a)
    mr = torch.empty((B, 2), dtype=torch.float32, device=a.device)
    scratch = torch.empty(160 * B, dtype=torch.float64, device=a.device)
    _check(lib.w2l_layernorm_fwd(_stream(), B, R, float(eps), _ptr(a), _ptr(r), _ptr(gain), _ptr(bias), _ptr(y), _ptr(mr),
                                 _ptr(scratch)))
    return y, mr


def layernorm_bwd(a, r, dy, gain, mr, branch_mode=0, branch_scale=1.0):
    B = a.shape[0]
    R = a[0].numel()
    d_branch = torch.empty_like(a)
    d_res = torch.empty_like(a)
    dgain = torch.zeros(1, dtype=torch.float32, device=a.device)
    dbias = torch.zeros(1, dtype=torch.float32, device=a.device)
    scratch = torch.empty(160 * B, dtype=torch.float64, device=a.device)
    _check(lib.w2l_layernorm_bwd(_stream(), B, R, _ptr(a), _ptr(r), _ptr(dy), _ptr(gain), _ptr(mr), _ptr(d_branch),
                                 _ptr(d_res), int(branch_mode), float(branch_scale), _ptr(dgain), _ptr(dbias),
                                 _ptr(scratch)))
    return d_branch, d_res, dgain, dbias


def soft_label_loss(student, teacher, scale=1.0, need_grad=True, d_student=None):
    """slimIPL's soft-label loss (w2l_soft_label_loss) over logits [..., N] (rows = every leading index): returns
    (loss float32 [1] = -scale / rows * sum_rows sum_c softmax(teacher)_c logSoftmax(student)_c,
    d_student = scale / rows * (softmax(student) - softmax(teacher)) or None).  d_student: an output buffer of the
    student's shape (any float alignment)."""
    student = _req(student, torch.float32, "student")
    teacher = _req(teacher, torch.float32, "teacher")
    if student.shape != teacher.shape:
        raise ValueError(f"soft_label_loss: teacher shape {tuple(teacher.shape)} != student shape {tuple(student.shape)}")
    N = student.shape[-1]
    rows = student.numel() // N
    loss = torch.empty(1, dtype=torch.float32, device=student.device)
    ws = torch.empty(rows, dtype=torch.float32, device=student.device)
    if need_grad and d_student is None:
        d_student = torch.empty_like(student)
    d = _req(d_student, torch.float32, "d_student") if need_grad else None
    _check(lib.w2l_soft_label_loss(_stream(), rows, N, _ptr(student), _ptr(teacher), float(scale), _ptr(loss), _ptr(d), _ptr(ws)))
    return loss, d


def ema_update(ema, params, decay):
    """in place: ema = ema * decay + params * (1 - decay) (w2l_ema_update), float32 tensors of the same size"""
    ema = _req(ema, torch.float32, "ema")
    params = _req(params, torch.float32, "params")
    if ema.numel() != params.numel():
        raise ValueError("ema_update: sizes differ")
    _check(lib.w2l_ema_update(_stream(), ema.numel(), _ptr(ema), _ptr(params), float(decay)))
    return ema
