# -*- coding: utf-8 -*-
"""ctypes binding of libwnb200.so (include/wnb200.h).

There is NO fallback: if the library is missing or a call fails, an exception is raised.
PyTorch is used only as the owner of device memory and streams; every pointer handed to the
library is ``tensor.data_ptr()`` and every launch goes to ``torch.cuda.current_stream()``.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libwnb200.so")

MATH_FP32 = 0
MATH_TF32 = 1
MATH_BF16 = 2
MODE_ARGMAX = 0
MODE_SAMPLING = 1

_c = ctypes
_P = _c.c_void_p
_I = _c.c_int
_L = _c.c_int64

# name -> (restype, argtypes); must list every symbol declared in include/wnb200.h
SIGNATURES = {
    "wnb_version": (_I, []),
    "wnb_last_error": (_c.c_char_p, []),
    "wnb_launch_count": (_L, []),
    "wnb_mulaw_encode_f32": (_I, [_P, _P, _L, _I, _P]),
    "wnb_mulaw_encode_f64": (_I, [_P, _P, _L, _I, _P]),
    "wnb_mulaw_decode_f64": (_I, [_P, _P, _L, _I, _P]),
    "wnb_lut_i16": (_I, [_P, _P, _P, _L, _I, _P]),
    "wnb_front_embed_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "wnb_front_embed_bwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "wnb_aux_upsample_fwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "wnb_aux_upsample_bwd": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "wnb_resblock_fwd": (_I, [_P] * 9 + [_I] * 9 + [_P]),
    "wnb_resblock_fwd_supported": (_I, [_I] * 5),
    "wnb_causal_conv1d_fwd": (_I, [_P] * 4 + [_I] * 6 + [_P]),
    "wnb_profile_enable": (_I, [_I]),
    "wnb_profile_read": (_I, [_I, _P, _P]),
    "wnb_wgrad_partition": (_I, [_P, _P, _P, _P, _I, _I, _P, _P, _I]),
    "wnb_wgrad_transpose_map": (_I, [_I, _P]),
    "wnb_stack_supported": (_I, [_I] * 6),
    "wnb_resblock_fwd_z": (_I, [_P] * 8 + [_I] * 8 + [_P]),
    "wnb_skip_gemm": (_I, [_P] * 4 + [_I] * 5 + [_P]),
    "wnb_stack_fwd": (_I, [_P, _I] + [_P] * 10 + [_I] * 8 + [_P]),
    "wnb_stack_bwd_workspace": (_c.c_size_t, [_I] * 7),
    "wnb_stack_bwd": (_I, [_P] * 19 + [_I] * 7 + [_P]),
    "wnb_resblock_bwd_workspace": (_c.c_size_t, [_I] * 6),
    "wnb_resblock_bwd": (_I, [_P] * 15 + [_I] * 8 + [_P]),
    "wnb_post_fwd": (_I, [_P] * 7 + [_I] * 6 + [_P]),
    "wnb_post_bwd": (_I, [_P] * 11 + [_I] * 5 + [_P]),
    "wnb_cross_entropy": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "wnb_cross_entropy_rows": (_I, [_P, _P, _P, _I, _P, _P, _I, _I, _I, _P]),
    "wnb_decode_workspace": (_c.c_size_t, [_I, _I, _I, _P, _I]),
    "wnb_decode_stream_floats": (_c.c_size_t, [_I] * 6),
    "wnb_decode_stream_supported": (_I, [_I] * 6),
    "wnb_decode_warp_floats": (_c.c_size_t, [_I, _I]),
    "wnb_decode_warp_set_timing": (None, [_P]),
    "wnb_decode_warp_supported": (_I, [_I] * 6),
    "wnb_decode_warp_plan": (_I, [_I]),
    "wnb_decode_warp_cluster": (_I, [_I]),
    "wnb_decode_warp_form": (_I, [_I, _I, _P]),
    "wnb_decode_bf16_supported": (_I, [_I] * 6),
    "wnb_decode_bf16_weights": (_c.c_size_t, [_I] * 6),
    "wnb_decode_bf16_workspace": (_c.c_size_t, [_I, _I, _I, _P, _I]),
    "wnb_decode_at": (_I, [_P] * 14 + [_P, _I] + [_P] * 4 + [_I] * 13 + [_c.c_uint64] + [_I] * 3 + [_P]),
    "wnb_decode_stream_at": (_I, [_P] * 11 + [_P, _I] + [_P] * 4 + [_I] * 13 + [_c.c_uint64] + [_I] * 3 + [_P]),
    "wnb_decode_warp_at": (_I, [_P] * 11 + [_P, _I] + [_P] * 4 + [_I] * 8 + [_c.c_uint64, _I, _I] + [_I] * 3 + [_P]),
    "wnb_decode_bf16_at": (_I, [_P] * 7 + [_P, _I] + [_P] * 4 + [_I] * 13 + [_c.c_uint64] + [_I] * 3 + [_P]),
    "wnb_decode_prefill_windows": (_I, [_P, _I, _I, _P]),
    "wnb_decode_prefill_workspace": (_c.c_size_t, [_I] * 4 + [_P, _I]),
    "wnb_decode_warp_prefill": (_I, [_P] * 11 + [_I] + [_P] * 2 + [_I] * 7 + [_P]),
    "wnb_decode_stream_prefill": (_I, [_P] * 9 + [_P, _I] + [_P] * 2 + [_I] * 11 + [_P]),
    "wnb_decode_bf16_prefill_workspace": (_c.c_size_t, [_I] * 4 + [_P, _I]),
    "wnb_decode_bf16_prefill": (_I, [_P] * 7 + [_P, _I] + [_P] * 2 + [_I] * 10 + [_P]),
    "wnb_decode_bf16_pool_transplant": (_I, [_P, _I, _P, _P, _I, _P, _P] + [_I] * 3 + [_P, _I, _P]),
    "wnb_decode_bf16_pool_inputs": (_I, [_P] * 6 + [_I] * 5 + [_c.c_uint64, _P]),
    "wnb_decode_bf16_park_bytes": (_c.c_size_t, [_I, _I, _P, _I]),
    "wnb_decode_bf16_pool_park": (_I, [_P, _I, _P, _P, _P] + [_I] * 3 + [_P, _I, _P]),
    "wnb_decode_bf16_pool_unpark": (_I, [_P, _P, _I, _P, _P] + [_I] * 3 + [_P, _I, _P]),
    "wnb_decode_pool_move": (_I, [_P, _P, _P] + [_I] * 3 + [_P, _I, _P]),
    "wnb_pack_weights": (_I, [_P, _I, _P, _P, _P, _P]),
    "wnb_zero": (_I, [_P, _c.c_size_t, _P]),
    "wnb_make_train_batch": (_I, [_P, _P, _P, _L, _L, _I, _L, _L] + [_P] * 5 + [_I] * 6 + [_P]),
    "wnb_make_train_batch_corpus": (_I, [_P] * 4 + [_I, _L, _L, _L, _L, _I] + [_P] * 5 + [_I] * 6 + [_P]),
    "wnb_adam_flat": (_I, [_P, _P, _P, _P, _L] + [_c.c_double] * 7 + [_P]),
    "wnb_mlsa_filter": (_I, [_P, _I, _P, _I, _P, _I, _c.c_double, _I, _c.c_double, _P, _I, _P]),
    "wnb_mlsa_state_doubles": (_c.c_size_t, [_I, _I]),
    "wnb_mlsa_filter_state": (_I, [_P, _I, _P, _I, _P, _I, _c.c_double, _I, _c.c_double, _P, _I, _P, _I, _P, _P, _P]),
    "wnb_melspc_lowcut": (_I, [_P, _I, _P, _I, _L, _P, _I, _P, _P, _P]),
    "wnb_melspc": (_I, [_P, _I, _P, _P, _I, _L, _I, _I] + [_P] * 5 + [_I, _P, _P]),
    "wnb_melspc_stream_state_doubles": (_c.c_size_t, [_I, _I]),
    "wnb_melspc_stream": (_I, [_P, _I, _I, _P, _P, _L, _I, _I, _P, _I] + [_P] * 5 + [_I, _P, _I, _P, _L, _P, _P, _P, _I,
                                                                                      _P, _P]),
    "wnb_mcep": (_I, [_P, _I, _P, _P, _I, _L, _I, _I, _I, _c.c_double] + [_P] * 5
                 + [_I, _I] + [_c.c_double] * 3 + [_P, _P, _P]),
    "wnb_mcd_aligned": (_I, [_P, _P, _I] + [_P] * 4 + [_I, _P, _P, _P]),
    "wnb_mcd_dtw_workspace": (_c.c_size_t, [_L, _L]),
    "wnb_mcd_dtw": (_I, [_P, _P, _I] + [_P] * 4 + [_I, _P, _c.c_size_t, _P, _P, _P, _P]),
}

_lib = None


def load():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libwnb200.so is missing (%s). Build it with `python -m pytorchwavenetvocoder_b200.build`; "
            "there is no CPU or PyTorch fallback for the hot path." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class WnbError(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        msg = load().wnb_last_error()
        raise WnbError("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))


def ptr(t):
    """Device pointer of a tensor (None -> NULL).  The tensor must be contiguous and on CUDA."""
    if t is None:
        return None
    if not t.is_cuda:
        raise WnbError("the wnb200 hot path needs CUDA tensors (got %s); there is no CPU fallback" % t.device)
    if not t.is_contiguous():
        raise WnbError("non-contiguous tensor handed to libwnb200")
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def launch_count():
    return int(load().wnb_launch_count())
