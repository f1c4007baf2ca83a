"""ctypes binding of the C-ABI library (include/torchbeast_b200.h).

There is NO fallback: if libtorchbeast_b200.so is missing, or a tensor is not on a CUDA
device, the call raises.  PyTorch is used only for device memory and streams.
"""
import ctypes
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libtorchbeast_b200.so")

_c = ctypes
_vp, _i64, _f32, _f64, _int = _c.c_void_p, _c.c_int64, _c.c_float, _c.c_double, _c.c_int

_SIGNATURES = {
    "tb_abi_version": ([], _int),
    "tb_last_error": ([], _c.c_char_p),
    "tb_device_info": ([_vp, _vp, _vp], _int),
    "tb_workspace_bytes": ([], _c.c_size_t),
    "tb_launch_count": ([], _c.c_uint64),
    "tb_profile_enable": ([_int], _int),
    "tb_profile_collect": ([_c.c_char_p, _c.c_size_t, _vp, _int], _int),
    "tb_action_log_probs_f32": ([_vp, _vp, _i64, _i64, _vp, _vp], _int),
    "tb_action_log_probs_f64": ([_vp, _vp, _i64, _i64, _vp, _vp], _int),
    "tb_vtrace_from_importance_weights_f32": ([_vp] * 5 + [_i64, _i64, _f32, _f32, _vp, _vp, _vp], _int),
    "tb_vtrace_from_importance_weights_f64": ([_vp] * 5 + [_i64, _i64, _f64, _f64, _vp, _vp, _vp], _int),
    "tb_hparams_layout": ([_vp], _int),
    "tb_impala_loss_f32": (
        [_vp] * 8 + [_i64, _i64, _i64, _f32, _f32, _f32, _int, _f32, _f32] + [_vp] * 5 + [_i64] + [_vp] * 12
        + [_int, _vp, _vp], _int),
    "tb_impala_loss_factored_f32": (
        [_vp] * 8 + [_i64, _i64, _i64, _f32, _f32, _f32, _int, _f32, _f32] + [_vp] * 5 + [_i64] + [_vp] * 12
        + [_int, _vp, _vp, _vp], _int),
    "tb_action_space_layout": ([_vp], _int),
    "tb_impala_loss_gaussian_f32": (
        [_vp] * 8 + [_i64, _i64, _i64, _f32, _f32, _f32, _int, _f32, _f32] + [_vp] * 5 + [_i64] + [_vp] * 12
        + [_int, _vp, _vp], _int),
    "tb_upgo_loss_f32": ([_vp] * 7 + [_i64, _i64, _i64, _f32, _int, _f32] + [_vp] * 5 + [_i64] + [_vp] * 10, _int),
    "tb_kickstart_loss_f32": ([_vp, _vp, _i64, _i64, _i64] + [_vp] * 7, _int),
    "tb_popart_update": ([_vp] * 4 + [_i64, _vp, _vp, _i64, _vp], _int),
    "tb_atarinet_param_count": ([_int, _int, _int], _i64),
    "tb_atarinet_workspace_bytes": ([_i64, _i64, _int, _int, _int], _c.c_size_t),
    "tb_atarinet_grad_split": ([_int, _int], _i64),
    "tb_atarinet_forward": ([_vp] * 8 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 7, _int),
    "tb_atarinet_forward_factored": ([_vp] * 8 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 8, _int),
    "tb_atarinet_backward": ([_vp] * 4 + [_i64, _i64, _int, _int, _int, _int, _vp, _vp, _int, _vp], _int),
    "tb_atarinet_param_count_continuous": ([_int, _int, _int], _i64),
    "tb_atarinet_workspace_bytes_continuous": ([_i64, _i64, _int, _int, _int], _c.c_size_t),
    "tb_atarinet_forward_continuous": ([_vp] * 8 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 7, _int),
    "tb_atarinet_backward_continuous": ([_vp] * 4 + [_i64, _i64, _int, _int, _int, _int, _vp, _vp, _int, _vp], _int),
    "tb_resnet_obs_range": ([_vp], _int),
    "tb_resnet_widths": ([_vp], _int),
    "tb_resnet_supported": ([_int] * 7, _int),
    "tb_resnet_param_count": ([_int] * 9, _i64),
    "tb_resnet_workspace_bytes": ([_int] * 6 + [_i64, _i64, _int, _int, _int], _c.c_size_t),
    "tb_resnet_forward": ([_vp] * 7 + [_int] * 6 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 7, _int),
    "tb_resnet_backward": ([_vp] * 5 + [_int] * 6 + [_i64, _i64, _int, _int, _int, _int, _vp, _vp, _vp], _int),
    "tb_sample_actions_f32": ([_vp, _i64, _i64, _i64, _c.c_uint64, _c.c_uint64, _vp, _vp, _vp], _int),
    "tb_sample_actions_dev_f32": ([_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_sample_actions_factored_f32": ([_vp, _i64, _i64, _i64, _c.c_uint64, _c.c_uint64] + [_vp] * 5, _int),
    "tb_sample_gaussian_f32": ([_vp, _i64, _i64, _i64, _c.c_uint64, _c.c_uint64] + [_vp] * 4, _int),
    "tb_mask_logits_f32": ([_vp, _vp, _vp, _vp, _i64, _i64, _f32, _vp], _int),
    "tb_replay_mix": ([_vp, _int, _i64, _i64, _i64, _vp, _vp, _i64, _vp, _vp], _int),
    "tb_replay_advance": ([_vp, _vp, _i64, _i64, _vp], _int),
    "tb_replay_mix_slots": ([_vp, _int, _i64, _i64, _i64, _vp, _vp, _vp], _int),
    "tb_replay_sample_prioritized": ([_vp] * 4 + [_i64, _i64, _i64, _i64, _vp, _vp, _vp], _int),
    "tb_replay_update_priorities": ([_vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_baseline_loss_f32": ([_vp, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_baseline_loss_f64": ([_vp, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_entropy_loss_f32": ([_vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_entropy_loss_f64": ([_vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_pg_loss_f32": ([_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_pg_loss_f64": ([_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_gemm_bf16_tn": ([_vp, _vp, _i64, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _i64, _vp, _f32, _int, _vp], _int),
    "tb_gemm_bf16_ex": ([_vp, _vp, _i64, _i64, _i64, _i64, _i64, _int, _int, _vp, _i64, _int, _vp, _vp], _int),
    "tb_gemm_bf16x3_ex": ([_vp, _vp, _i64, _i64, _i64, _i64, _i64, _int, _int, _i64, _i64, _vp, _i64, _vp, _i64, _i64, _vp,
                           _f32, _int, _vp, _i64, _int, _vp, _vp], _int),
    "tb_conv_nhwc_bf16_fwd": ([_vp, _vp, _vp, _i64] + [_int] * 8 + [_vp, _vp, _vp], _int),
    "tb_conv_nhwc_bf16_dgrad": ([_vp, _vp, _vp, _i64] + [_int] * 7 + [_vp, _vp, _vp], _int),
    "tb_conv_nhwc_bf16_wgrad": ([_vp, _vp, _i64] + [_int] * 7 + [_vp, _vp, _i64, _vp], _int),
    "tb_conv1_u8_fwd": ([_vp, _vp, _vp, _i64, _int, _int, _int, _int, _vp, _vp, _vp, _vp], _int),
    "tb_conv1_u8_wgrad": ([_vp, _vp, _i64, _int, _int, _int, _vp, _vp, _i64, _vp], _int),
    "tb_conv_nhwc_bf16x3_fwd": ([_vp, _i64, _vp, _vp, _i64] + [_int] * 8 + [_vp, _i64, _vp, _vp], _int),
    "tb_conv_nhwc_bf16x3_dgrad": ([_vp, _i64, _vp, _vp, _i64] + [_int] * 7 + [_vp, _i64, _vp, _vp], _int),
    "tb_conv_nhwc_bf16x3_wgrad": ([_vp, _i64, _vp, _i64, _i64] + [_int] * 7 + [_vp, _vp, _i64, _vp], _int),
    "tb_conv1_u8_bf16x3_fwd": ([_vp, _vp, _vp, _i64, _int, _int, _int, _int, _vp, _i64, _vp, _vp, _vp], _int),
    "tb_conv1_u8_bf16x3_wgrad": ([_vp, _i64, _vp, _i64, _int, _int, _int, _vp, _vp, _i64, _vp], _int),
    "tb_sw_image_elems": ([_i64, _int, _int, _int], _i64),
    "tb_sw_pad_split_f32": ([_vp, _vp, _i64, _i64, _int, _int, _int, _int, _vp, _vp, _i64, _vp], _int),
    "tb_sw_colsum_scratch_floats": ([_i64, _int, _int, _int], _i64),
    "tb_sw_frames_u8": ([_vp, _vp, _i64, _i64, _int, _int, _int, _vp], _int),
    "tb_sw_weight_elems": ([_int, _int], _i64),
    "tb_sw_pack_weights": ([_vp, _vp, _int, _int, _int, _int, _vp], _int),
    "tb_sw_conv_fwd": ([_vp, _i64, _vp, _vp, _i64, _int, _int, _int, _int, _f32, _vp, _vp, _vp, _vp, _i64, _int, _vp, _vp],
                       _int),
    "tb_sw_csum_rows": ([_i64, _int, _int], _i64),
    "tb_sw_csum_reduce": ([_vp, _i64, _int, _vp, _vp], _int),
    "tb_sw_conv_wgrad": ([_vp, _i64, _vp, _i64, _vp, _i64, _int, _int, _int, _int, _f32, _int, _vp, _i64, _vp], _int),
    "tb_sw_pool_bwd_image_colsum": ([_vp, _vp, _vp, _i64, _i64, _int, _int, _int, _vp, _vp, _i64, _vp], _int),
    "tb_maxpool3x3s2_fwd_f32": ([_vp, _vp, _vp, _i64, _int, _int, _int, _vp], _int),
    "tb_f32_to_bf16": ([_vp, _vp, _i64, _i64, _i64, _i64, _vp], _int),
    "tb_gemm_f32": ([_vp, _int, _vp, _int, _int, _int] + [_i64] * 5 + [_vp, _i64, _vp, _int, _vp, _i64, _vp, _i64, _int, _int,
                                                                        _int, _f32, _int, _vp, _vp], _int),
    "tb_gemm_f32_splits": ([_i64] * 5, _int),
    "tb_splitk_scratch_floats": ([], _i64),
    "tb_im2col_u8_nchw": ([_vp, _vp, _i64] + [_int] * 6 + [_vp], _int),
    "tb_im2col_f32_nhwc": ([_vp, _vp, _i64] + [_int] * 6 + [_vp], _int),
    "tb_col2im_f32_nhwc": ([_vp, _vp, _vp, _i64] + [_int] * 6 + [_vp], _int),
    "tb_permute_pq": ([_vp, _vp, _i64, _int, _int, _vp], _int),
    "tb_relu_mask_f32": ([_vp, _vp, _i64, _i64, _i64, _i64, _vp], _int),
    "tb_core_extras": ([_vp, _i64, _i64, _int, _vp, _vp, _int, _vp], _int),
    "tb_im2col3x3": ([_vp, _vp, _i64, _int, _int, _int, _i64, _int, _int, _vp], _int),
    "tb_im2col3x3_u8": ([_vp, _vp, _i64, _int, _int, _int, _i64, _int, _vp], _int),
    "tb_col2im3x3": ([_vp, _vp, _vp, _vp, _i64, _int, _int, _int, _i64, _int, _vp], _int),
    "tb_maxpool3x3s2_fwd": ([_vp, _vp, _vp, _i64, _int, _int, _int, _int, _vp], _int),
    "tb_maxpool3x3s2_bwd": ([_vp, _vp, _vp, _i64, _int, _int, _int, _int, _vp], _int),
    "tb_relu_fwd": ([_vp, _vp, _i64, _int, _vp], _int),
    "tb_relu_bwd": ([_vp, _vp, _vp, _i64, _int, _vp], _int),
    "tb_colsum_scratch_floats": ([_i64], _i64),
    "tb_colsum_f32": ([_vp, _vp, _i64, _i64, _i64, _vp, _vp], _int),
    "tb_colsum_bf16": ([_vp, _vp, _i64, _i64, _i64, _vp, _i64, _vp], _int),
    "tb_heads_scratch_floats": ([_i64, _int, _int, _int], _i64),
    "tb_heads_forward": ([_vp, _i64, _vp, _vp, _vp, _vp, _i64, _int, _int, _int, _vp, _vp, _vp], _int),
    "tb_heads_backward": ([_vp, _i64, _vp, _vp, _vp, _vp, _i64, _int, _int, _int, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp],
                          _int),
    "tb_grad_sumsq_f32": ([_vp, _i64, _vp, _vp, _vp], _int),
    "tb_clip_rmsprop_step_f32": ([_vp] * 4 + [_i64, _vp, _f32, _vp, _f32, _f32, _f32, _f32, _vp, _vp, _vp], _int),
    "tb_clip_adam_step_f32": (
        [_vp] * 4 + [_i64, _vp, _f32, _vp, _f32, _f64, _f64, _f32, _f32, _int, _vp, _vp, _vp, _vp], _int),
    "tb_clip_rmsprop_ex_step_f32": (
        [_vp] * 5 + [_i64, _vp, _f32, _vp, _f32, _f32, _f32, _f32, _f32, _vp, _vp, _vp], _int),
    "tb_set_aux_stream": ([_vp], _int),
    "tb_restack_frames_u8": ([_vp, _vp, _i64, _i64, _i64, _vp, _vp], _int),
    "tb_frame_history_fill_u8": ([_vp, _vp, _vp, _i64, _i64, _i64, _vp, _i64, _vp], _int),
    "tb_unstacked_scratch_bytes": ([_int, _i64, _i64, _int], _c.c_size_t),
    "tb_host_write_rollout_column": ([_vp, _vp, _vp, _int, _i64, _i64, _i64, _vp], _int),
    "tb_lstm_workspace_bytes": ([_i64, _i64, _int, _int, _int, _int], _c.c_size_t),
    "tb_lstm_plan": ([_i64, _int, _int, _int, _int, _vp, _vp], _int),
    "tb_lstm_plan_layers": ([_i64, _int, _int, _int, _int, _vp, _vp], _int),
    "tb_lstm_forward": ([_vp] * 5 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 5, _int),
    "tb_lstm_backward": ([_vp] * 5 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 3, _int),
    "tb_lstm_backward_state": ([_vp] * 5 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 7, _int),
}

_lib = None
_lock = threading.Lock()


class TorchBeastB200Error(RuntimeError):
    pass


def declared_symbols():
    """Every entry point include/torchbeast_b200.h declares (kept in sync by tests)."""
    return sorted(_SIGNATURES)


def lib():
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise ImportError(
                        "torchbeast_b200: %s not found. Build it with `python -c 'import __graft_entry__ as g; "
                        "g.build()'` (nvcc, sm_90a). There is no CPU/PyTorch fallback." % LIB_PATH)
                h = ctypes.CDLL(LIB_PATH)
                for name, (argtypes, restype) in _SIGNATURES.items():
                    fn = getattr(h, name)  # AttributeError if the .so lacks a declared symbol
                    fn.argtypes = argtypes
                    fn.restype = restype
                if h.tb_abi_version() != 1:
                    raise ImportError("torchbeast_b200: ABI version mismatch")
                _lib = h
    return _lib


def check(rc, what):
    if rc != 0:
        raise TorchBeastB200Error("%s failed (%d): %s" % (what, rc, lib().tb_last_error().decode()))


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise TorchBeastB200Error(
                "torchbeast_b200 runs on CUDA tensors only (got a %s tensor); there is no CPU fallback - "
                "use the reference implementation for CPU work." % t.device)


_workspaces = {}


def workspace():
    """Zero-initialised scratch for the reducing kernels, one per (device, stream)."""
    key = (torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)
    ws = _workspaces.get(key)
    if ws is None:
        ws = torch.zeros(lib().tb_workspace_bytes(), dtype=torch.uint8, device="cuda")
        _workspaces[key] = ws
    return ws


def clip_arg(c):
    return -1.0 if c is None else float(c)


def profile_collect(max_records=65536):
    """Return [(op_name, milliseconds), ...] recorded since tb_profile_enable(1)."""
    names = ctypes.create_string_buffer(max_records * 48)
    ms = (ctypes.c_float * max_records)()
    n = lib().tb_profile_collect(names, len(names), ctypes.cast(ms, ctypes.c_void_p), max_records)
    if n < 0:
        raise TorchBeastB200Error("tb_profile_collect failed: %s" % lib().tb_last_error().decode())
    nm = names.value.decode().split("\n")[:n]
    return list(zip(nm, [ms[i] for i in range(n)]))
