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
    "tb_impala_loss_fwd_bwd_f32": (
        [_vp] * 8 + [_i64, _i64, _i64, _f32, _f32, _f32, _int, _f32, _f32] + [_vp] * 8 + [_int, _vp, _vp], _int),
    "tb_sample_actions_f32": ([_vp, _i64, _i64, _i64, _c.c_uint64, _c.c_uint64, _vp, _vp, _vp], _int),
    "tb_sample_actions_dev_f32": ([_vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_baseline_loss_f32": ([_vp, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_baseline_loss_f64": ([_vp, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_entropy_loss_f32": ([_vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_entropy_loss_f64": ([_vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_pg_loss_f32": ([_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_pg_loss_f64": ([_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp], _int),
    "tb_gemm_bf16_tn": ([_vp, _vp, _i64, _i64, _i64, _i64, _i64, _vp, _i64, _vp, _i64, _vp, _f32, _int, _vp], _int),
    "tb_gemm_bf16_ex": ([_vp, _vp, _i64, _i64, _i64, _i64, _i64, _int, _int, _vp, _i64, _int, _vp, _vp], _int),
    "tb_conv_nhwc_bf16_fwd": ([_vp, _vp, _vp, _i64] + [_int] * 8 + [_vp, _vp, _vp], _int),
    "tb_conv_nhwc_bf16_dgrad": ([_vp, _vp, _vp, _i64] + [_int] * 7 + [_vp, _vp, _vp], _int),
    "tb_conv_nhwc_bf16_wgrad": ([_vp, _vp, _i64] + [_int] * 7 + [_vp, _vp, _i64, _vp], _int),
    "tb_conv1_u8_fwd": ([_vp, _vp, _vp, _i64, _int, _int, _int, _int, _vp, _vp, _vp, _vp], _int),
    "tb_conv1_u8_wgrad": ([_vp, _vp, _i64, _int, _int, _int, _vp, _vp, _i64, _vp], _int),
    "tb_f32_to_bf16": ([_vp, _vp, _i64, _i64, _i64, _i64, _vp], _int),
    "tb_atarinet_param_count": ([_int, _int], _i64),
    "tb_atarinet_workspace_bytes": ([_i64, _i64, _int, _int, _int], _c.c_size_t),
    "tb_atarinet_forward": ([_vp] * 7 + [_i64, _i64, _int, _int, _int] + [_vp] * 6, _int),
    "tb_resnet_param_count": ([_int, _int], _i64),
    "tb_resnet_workspace_bytes": ([_i64, _i64, _int, _int, _int], _c.c_size_t),
    "tb_resnet_forward": ([_vp] * 6 + [_i64, _i64, _int, _int, _int] + [_vp] * 6, _int),
    "tb_resnet_backward": ([_vp] * 5 + [_i64, _i64, _int, _int, _int, _vp, _vp, _vp], _int),
    "tb_grad_sumsq_f32": ([_vp, _i64, _vp, _vp, _vp], _int),
    "tb_clip_rmsprop_step_f32": ([_vp] * 4 + [_i64, _vp, _f32, _vp, _f32, _f32, _f32, _f32, _vp, _vp], _int),
    "tb_atarinet_backward": ([_vp] * 4 + [_i64, _i64, _int, _int, _int, _vp, _vp, _vp], _int),
    "tb_atarinet_grad_split": ([_int, _int], _i64),
    "tb_set_aux_stream": ([_vp], _int),
    "tb_host_write_rollout_column": ([_vp, _vp, _vp, _int, _i64, _i64, _i64, _vp], _int),
    "tb_lstm_workspace_bytes": ([_i64, _i64, _int, _int, _int, _int], _c.c_size_t),
    "tb_lstm_forward": ([_vp] * 5 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 5, _int),
    "tb_lstm_backward": ([_vp] * 5 + [_i64, _i64, _int, _int, _int, _int] + [_vp] * 3, _int),
    "tb_atarinet_backward_phase": ([_vp] * 4 + [_i64, _i64, _int, _int, _int, _vp, _vp, _int, _vp], _int),
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
