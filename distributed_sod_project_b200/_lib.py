"""ctypes binding of libsod_b200.so (C ABI in include/sod_b200.h).

There is deliberately NO fallback: if the library is missing or a call fails, the hot path raises.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsod_b200.so")

SOD_F32, SOD_BF16, SOD_F16 = 0, 1, 2
SOD_MAX_WORLD = 8
SOD_MAX_SEGMENTS = 16
SOD_SEG_FROZEN = 1
SOD_SEG_GRAD16 = 2
SOD_SEG_NESTEROV = 4
SOD_SGD_ZERO_GRAD = 1
SOD_ALGO_NO_MULTIMEM = 2
SOD_BN_ACCUMULATE_PARAM_GRADS = 8
SOD_ALGO_FORCE_MULTIMEM = 16
SOD_BN_BWD_MASK_FROM_X = 32
SOD_BN_L2_HINTS = 64
SOD_BN_LAUNCH_COOP = 128
SOD_BN_LAUNCH_PDL = 256
SOD_GRAD16_F16 = 512
SOD_GN_GROUPS = 32
SOD_GCONV_GROUPS = 32
SOD_RESIZE_BILINEAR = 2
SOD_RESIZE_BICUBIC = 3
SOD_GATHER_MAX_ITEMS = 160
SOD_CHECK_MAX_RANGES = 128
SOD_ADAM_STEP_WORDS = SOD_MAX_SEGMENTS + 1
ABI_VERSION = 7


class SodError(RuntimeError):
    pass


class sod_comm(C.Structure):
    _fields_ = [("rank", C.c_int32), ("world", C.c_int32), ("peer", C.c_uint64 * SOD_MAX_WORLD),
                ("mc", C.c_uint64), ("arena_bytes", C.c_uint64), ("error_flag", C.c_void_p),
                ("timeout_cycles", C.c_uint64), ("block_seq", C.c_void_p)]


class sod_gather_item(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst_offset", C.c_int64), ("numel", C.c_int64)]


class sod_sgd_segment(C.Structure):
    _fields_ = [("begin", C.c_int64), ("end", C.c_int64), ("lr", C.c_float), ("weight_decay", C.c_float),
                ("momentum", C.c_float), ("flags", C.c_int32)]


class sod_adam_segment(C.Structure):
    _fields_ = [("begin", C.c_int64), ("end", C.c_int64), ("lr", C.c_float), ("weight_decay", C.c_float),
                ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("flags", C.c_int32)]


class sod_loss_scaler(C.Structure):
    _fields_ = [("found_inf", C.c_uint32), ("scale", C.c_float), ("unskipped", C.c_int32), ("growth_interval", C.c_int32),
                ("ticket", C.c_uint32), ("reserved", C.c_uint32 * 3)]


SOD_LOSS_SCALER_WORDS = 8     # sizeof(sod_loss_scaler) / 4: [found_inf, scale (fp32 bits), unskipped, growth_interval, ticket, …]


class sod_check_range(C.Structure):
    _fields_ = [("begin", C.c_int64), ("end", C.c_int64), ("flags", C.c_int32)]


class sod_augment_param(C.Structure):
    _fields_ = [("rot", C.c_double * 6), ("flip", C.c_int32), ("identity", C.c_int32), ("ops", C.c_int32 * 3),
                ("factor", C.c_float * 3)]


_PROTOTYPES = {
    "sod_version": (C.c_int, []),
    "sod_strerror": (C.c_char_p, [C.c_int]),
    "sod_device_info": (C.c_int, [C.POINTER(C.c_int)] * 3),
    "sod_loss_workspace_bytes": (C.c_size_t, []),
    "sod_loss_bce_cel_fwd_bwd": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                           C.c_int64, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int,
                                           C.c_void_p, C.c_size_t, C.c_void_p]),
    "sod_loss_bce_cel_fwd_bwd_scaled": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                                  C.c_int64, C.c_int, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_float,
                                                  C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sod_scale_by_device_scalar": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p]),
    "sod_comm_flag_bytes": (C.c_size_t, []),
    "sod_sgd_momentum": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                   C.POINTER(sod_sgd_segment), C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_void_p]),
    "sod_allreduce_sgd": (C.c_int, [C.POINTER(sod_comm), C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_int64,
                                    C.POINTER(sod_sgd_segment), C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_int, C.c_void_p]),
    "sod_adam": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                           C.POINTER(sod_adam_segment), C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int,
                           C.c_void_p]),
    "sod_allreduce_adam": (C.c_int, [C.POINTER(sod_comm), C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_int64, C.POINTER(sod_adam_segment), C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_float, C.c_void_p, C.c_int, C.c_void_p]),
    "sod_sgd_momentum_scaler": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                          C.POINTER(sod_sgd_segment), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "sod_allreduce_sgd_scaler": (C.c_int, [C.POINTER(sod_comm), C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                           C.c_int64, C.POINTER(sod_sgd_segment), C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                           C.c_void_p]),
    "sod_adam_scaler": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                  C.POINTER(sod_adam_segment), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "sod_allreduce_adam_scaler": (C.c_int, [C.POINTER(sod_comm), C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int64, C.POINTER(sod_adam_segment), C.c_int, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int, C.c_void_p]),
    "sod_grad_gather16": (C.c_int, [C.POINTER(sod_gather_item), C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "sod_grad_gather16_checked": (C.c_int, [C.POINTER(sod_gather_item), C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p,
                                            C.c_void_p]),
    "sod_grad_merge_bf16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "sod_grad_merge16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "sod_grad_nonfinite": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]),
    "sod_grad_check_ranges": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(sod_check_range), C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p]),
    "sod_allreduce_f32": (C.c_int, [C.POINTER(sod_comm), C.c_uint64, C.c_int64, C.c_float, C.c_int, C.c_int, C.c_void_p]),
    "sod_syncbn_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int]),
    "sod_syncbn_exchange_bytes": (C.c_size_t, [C.c_int]),
    "sod_syncbn_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_float, C.c_float,
                                 C.c_int, C.c_int, C.POINTER(sod_comm), C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "sod_syncbn_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int,
                                 C.POINTER(sod_comm), C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "sod_upsample2x_bilinear_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sod_upsample2x_bilinear_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sod_avgpool2x2_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sod_avgpool2x2_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sod_colsum_workspace_bytes": (C.c_size_t, []),
    "sod_colsum": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sod_maxpool3x3s2_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sod_preprocess_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p]),
    "sod_saliency_quantize": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "sod_saliency_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "sod_saliency_hist": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sod_maxpool3x3s2_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sod_maxpool2x2s2_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sod_maxpool2x2s2_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "sod_saliency_head_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sod_saliency_hist_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p]),
    "sod_saliency_wfm_workspace_bytes": (C.c_size_t, [C.c_int, C.c_void_p]),
    "sod_saliency_wfm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sod_saliency_wfm_ragged": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    "sod_resize_u8_workspace_bytes":(C.c_size_t, [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]),
    "sod_resize_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sod_augment_u8_workspace_bytes": (C.c_size_t, [C.c_int]),
    "sod_augment_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(sod_augment_param),
                                 C.c_void_p, C.c_size_t, C.c_void_p]),
    "sod_groupnorm_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int, C.c_int]),
    "sod_groupnorm_splits": (C.c_int, [C.c_int, C.c_int64, C.c_int, C.c_int]),
    "sod_groupnorm_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_int64, C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "sod_groupnorm_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                    C.c_int, C.c_void_p]),
    "sod_ws_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "sod_ws_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_void_p]),
    "sod_gconv3x3_fwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_int, C.c_void_p]),
    "sod_gconv3x3_dgrad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p]),
    "sod_gconv3x3_wgrad_splits": (C.c_int, [C.c_int] * 6),
    "sod_gconv3x3_wgrad_workspace_bytes": (C.c_size_t, [C.c_int] * 6),
    "sod_gconv3x3_wgrad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
}

EXPORTS = tuple(_PROTOTYPES)
_lib = None
_lock = threading.Lock()
launches = 0   # number of kernel-launching C-ABI calls made by this process (bench.py reports it)
grad_writes = 0   # bumped whenever a kernel of this library adds into a bound .grad (invisible to autograd's version counters)


def lib() -> C.CDLL:
    """Load (once) and return the shared library; raises SodError if it has not been built."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise SodError(f"{LIB_PATH} is missing: run `python -m distributed_sod_project_b200.build` "
                                   "(the CUDA hot path has no fallback)")
                h = C.CDLL(LIB_PATH)
                for name, (res, args) in _PROTOTYPES.items():
                    fn = getattr(h, name)
                    fn.restype, fn.argtypes = res, args
                _lib = h
    return _lib


def check(code: int, what: str = "") -> None:
    if code != 0:
        msg = lib().sod_strerror(code).decode()
        raise SodError(f"{what or 'libsod_b200'} failed: [{code}] {msg}")


def dtype_code(dtype) -> int:
    import torch
    try:
        return {torch.float32: SOD_F32, torch.bfloat16: SOD_BF16, torch.float16: SOD_F16}[dtype]
    except KeyError:
        raise SodError(f"unsupported dtype {dtype}") from None


def stream_ptr() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


def count_launch(n: int = 1) -> None:
    global launches
    launches += n
