"""ctypes binding of libb200asr.so (the C ABI declared in include/b200asr.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``build.sh``.  There is no fallback of any
kind: if the shared object is missing, or the device is not an sm_90 part (H100), importing callers get a
RuntimeError that says so.
"""
from __future__ import annotations

import ctypes as C
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200ASR_LIB", os.path.join(_HERE, "libb200asr.so"))   # override: A/B builds of the same ABI
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "b200asr.h")

_lib = None

PREC_FP32, PREC_TF32, PREC_TF32X3 = 0, 1, 3
PREC_BF16, PREC_BF16X3 = 2, 6          # bf16 modes (include/b200asr.h)

_vp, _i, _f, _u64, _ll, _sz = C.c_void_p, C.c_int, C.c_float, C.c_uint64, C.c_longlong, C.c_size_t

# name -> (restype, argtypes); every symbol declared in include/b200asr.h appears here
SIGNATURES = {
    "b200asr_version": (_i, []),
    "b200asr_last_error": (C.c_char_p, []),
    "b200asr_device_check": (_i, []),
    "b200asr_launch_count": (C.c_ulonglong, []),
    "b200asr_linear_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "b200asr_linear_bwd_data": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "b200asr_split_tf32": (_i, [_vp, _vp, _ll, _vp]),
    "b200asr_split_bf16": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "b200asr_split_bf16_batched": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp]),
    "b200asr_linear_bwd_weight": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200asr_add_ln_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _f, _f, _u64, _u64, _vp]),
    "b200asr_add_ln_bwd": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _f, _u64, _u64, _i, _vp]),
    "b200asr_add_ln_bwd_ws_bytes": (_sz, [_i, _i]),
    "b200asr_sdpa_fwd": (_i, [_vp, _vp, _vp] + [_ll] * 9 + [_vp, _vp, _i, _vp, _ll, _ll, _ll, _vp] + [_i] * 6 +
                         [_f, _f, _u64, _u64, _i, _vp]),
    "b200asr_sdpa_bwd": (_i, [_vp] * 6 + [_ll] * 12 + [_vp, _vp, _i, _vp, _vp, _vp, _vp] + [_i] * 6 +
                         [_f, _f, _u64, _u64, _i, _vp]),
    "b200asr_sdpa_fused_ws_bytes": (_sz, [_i, _i, _i, _i]),
    "b200asr_sdpa_fused_bwd_ws_bytes": (_sz, [_i, _i, _i]),
    "b200asr_sdpa_fused_fwd": (_i, [_vp, _vp, _vp] + [_ll] * 9 + [_vp, _vp, _i, _vp, _ll, _ll, _ll, _vp, _vp] + [_i] * 6 +
                               [_f, _f, _u64, _u64, _vp]),
    "b200asr_sdpa_fused_bwd": (_i, [_vp] * 6 + [_ll] * 12 + [_vp, _vp, _i, _vp, _vp, _vp, _vp, _vp] + [_i] * 6 +
                               [_f, _f, _u64, _u64, _vp]),
    "b200asr_sdpa_probs": (_i, [_vp, _vp] + [_ll] * 6 + [_vp, _vp, _i, _vp, _vp, _ll, _ll, _ll] + [_i] * 5 +
                           [_f, _f, _u64, _u64, _i, _vp]),
    "b200asr_sdpa_mat_ws_bytes": (_sz, [_i, _i, _i, _i]),
    "b200asr_sdpa_mat_fwd": (_i, [_vp, _vp, _vp] + [_ll] * 9 + [_vp, _vp, _i, _vp, _ll, _ll, _ll, _vp, _vp] + [_i] * 6 +
                             [_f, _f, _u64, _u64, _i, _vp]),
    "b200asr_sdpa_mat_bwd": (_i, [_vp] * 4 + [_ll] * 12 + [_vp] * 6 + [_i] * 6 + [_f, _f, _u64, _u64, _i, _vp]),
    "b200asr_stft_ws_bytes": (_sz, [_i, _i, _i, _i]),
    "b200asr_stft_features": (_i, [_vp] * 5 + [_i] * 9 + [_vp]),
    "b200asr_stft_features_ex_ws_bytes": (_sz, [_i, _i, _i, _i]),
    "b200asr_stft_features_ex": (_i, [_vp] * 5 + [_i] * 9 + [_vp, _ll, _vp, _vp, _i, _i, _vp]),
    "b200asr_stft_features_packed": (_i, [_vp] * 6 + [_i] * 9 + [_vp, _ll, _vp, _vp, _i, _i, _vp]),
    "b200asr_conv3x3_c1_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200asr_conv3x3_c1_bwd_weight": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "b200asr_conv3x3_fwd": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "b200asr_conv3x3_fwd_pool": (_i, [_vp] * 7 + [_i] * 7 + [_vp]),
    "b200asr_maxpool2x2_fwd_idx": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "b200asr_maxpool2x2_bwd_idx": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200asr_conv3x3_bwd_data": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200asr_conv3x3_c1_fwd_bits": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "b200asr_conv3x3_fwd_bits": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "b200asr_conv3x3_bwd_data_bits": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200asr_conv3x3_fwd_pool_codes": (_i, [_vp] * 7 + [_i] * 7 + [_vp]),
    "b200asr_maxpool2x2_bwd_codes": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200asr_conv3x3_bwd_weight": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "b200asr_conv3x3_ws_bytes": (_sz, [_i, _i]),
    "b200asr_maxpool2x2_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "b200asr_maxpool2x2_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200asr_conv2d_fwd": (_i, [_vp, _vp, _vp, _vp] + [_i] * 11 + [_vp]),
    "b200asr_conv2d_bwd_data": (_i, [_vp, _vp, _vp] + [_i] * 11 + [_vp]),
    "b200asr_conv2d_bwd_weight": (_i, [_vp, _vp, _vp, _vp] + [_i] * 11 + [_vp]),
    "b200asr_bn_ws_bytes": (_sz, [_i]),
    "b200asr_bn_clamp_fwd": (_i, [_vp] * 10 + [_i] * 6 + [_f, _f, _i, _f, _f, _vp]),
    "b200asr_bn_clamp_bwd": (_i, [_vp] * 10 + [_i] * 9 + [_f, _f, _vp]),
    "b200asr_conv2d_tc_ws_bytes": (_sz, [_i] * 5),
    "b200asr_conv2d_c1_tc_ws_bytes": (_sz, [_i] * 5),
    "b200asr_conv2d_c1_tc_fwd": (_i, [_vp] * 5 + [_i] * 9 + [_vp]),
    "b200asr_conv2d_c1_tc_bwd_weight": (_i, [_vp] * 5 + [_i] * 8 + [_vp]),
    "b200asr_conv2d_tc_fwd": (_i, [_vp] * 5 + [_i] * 11 + [_vp]),
    "b200asr_conv2d_tc_bwd_data": (_i, [_vp] * 4 + [_i] * 11 + [_vp]),
    "b200asr_conv2d_tc_bwd_weight": (_i, [_vp] * 5 + [_i] * 10 + [_vp]),
    "b200asr_flatten_bcft_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "b200asr_flatten_bcft_bwd": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "b200asr_preprocess_targets": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    "b200asr_embed_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _f, _u64, _u64, _vp]),
    "b200asr_embed_bwd": (_i, [_vp, _vp, _vp, _i, _i, _i, _f, _f, _u64, _u64, _i, _vp]),
    "b200asr_length_masks": (_i, [_vp, _vp, _vp, _i, _i, _vp]),
    "b200asr_argmax_rows": (_i, [_vp, _vp, _i, _i, _vp]),
    "b200asr_greedy_step": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "b200asr_beam_step": (_i, [_vp, _vp] + [_i] * 7 + [C.c_double, _vp, _vp, _vp, _vp, _vp, _i] + [_vp] * 7 + [_vp]),
    "b200asr_beam_self_attn": (_i, [_vp] * 5 + [_i] * 7 + [_f, _vp]),
    "b200asr_beam_backtrack": (_i, [_vp] * 6 + [_i] * 4 + [_vp]),
    "b200asr_decode_attn_ws_bytes": (_sz, [_i] * 4),
    "b200asr_decode_attn": (_i, [_vp] * 5 + [_i] * 5 + [_ll] * 4 + [_f, _vp]),
    "b200asr_beam_step_log": (_i, [_vp, _vp] + [_i] * 7 + [C.c_double, _vp, _vp, _vp, _vp, _vp, _i] + [_vp] * 7 + [_vp] * 3 +
                              [_i, _vp]),
    "b200asr_beam_backtrack_packed": (_i, [_vp] * 4 + [_i, _vp, _vp, _i, _vp, _i, _i, _i, _vp]),
    "b200asr_lstm_prepare": (_i, [_vp] * 4 + [_i, _i] + [_vp] * 3 + [_vp]),
    "b200asr_lstm_layer_fwd": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "b200asr_lstm_layer_train_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "b200asr_lstm_layer_train_bwd": (_i, [_vp] * 7 + [_i, _i, _i] + [_vp] * 4),
    "b200asr_lstm_dropout": (_i, [_vp, _vp, _ll, _f, _u64, _u64, _vp]),
    "b200asr_lstm_grad_unprepare": (_i, [_vp] * 3 + [_i, _i] + [_vp] * 5),
    "b200asr_lm_nll": (_i, [_vp, _ll, _vp, _vp, _i, _i, _vp]),
    "b200asr_lm_seq_sum": (_i, [_vp, _vp, _vp, _i, _vp, _vp]),
    "b200asr_xent_fwd": (_i, [_vp, _ll, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    "b200asr_xent_bwd": (_i, [_vp, _ll, _vp, _vp, _vp, _vp, _i, _i, _vp]),
    "b200asr_ce_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "b200asr_ce_finalize": (_i, [_vp, _vp, _i, _vp]),
    "b200asr_ce_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _f, _vp, _vp, _vp]),
    "b200asr_ctc_ws_bytes": (_sz, [_i, _i, _i]),
    "b200asr_ctc_fwd": (_i, [_vp] * 7 + [_i] * 5 + [_vp]),
    "b200asr_ctc_bwd": (_i, [_vp] * 8 + [_i] * 5 + [_vp]),
    "b200asr_adam_step": (_i, [_vp, _vp, _vp, _vp, _ll, _f, _f, _f, _f, _i, _f, _vp, _vp]),
    "b200asr_sumsq": (_i, [_vp, _ll, _vp, _vp]),
    "b200asr_grad_scale": (_i, [_vp, _ll, _vp, _f, _vp, _vp, _vp]),
    "b200asr_optim_table_capacity": (_i, []),
    "b200asr_adam_multi": (_i, [_vp, _vp, _vp, _vp, _i, _f, _f, _f, _f, _vp]),
    "b200asr_norm_multi": (_i, [_vp, _vp, _i, _vp, _vp]),
    "b200asr_clip_coef": (_i, [_vp, _i, _f, _vp, _vp]),
    "b200asr_scale_multi": (_i, [_vp, _vp, _i, _vp, _vp]),
    "b200asr_sgd_multi": (_i, [_vp, _vp, _i, _f, _vp]),
    "b200asr_permute_cols_cf":(_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "b200asr_edit_counts_ws_bytes": (_sz, [_i, _i, _i, _i]),
    "b200asr_edit_counts": (_i, [_vp, _i, _ll, _i, _vp, _i, _ll, _i, _i] + [_vp] * 5 + [_i, _i, _ll, _vp, _vp, _vp, _vp]),
}


def header_symbols():
    """Names of every function declared in include/b200asr.h (used by the ABI tests)."""
    with open(HEADER_PATH) as f:
        text = f.read()
    return sorted(set(re.findall(r"\b(b200asr_[a-z0-9_]+)\s*\(", text)))


def load(check_device: bool = False):
    """dlopen the in-tree library and attach prototypes.  Raises RuntimeError if it was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or ./build.sh).  There is no CPU or PyTorch fallback for this path.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    if check_device:
        rc = _lib.b200asr_device_check()
        if rc != 0:
            raise RuntimeError("libb200asr: " + _lib.b200asr_last_error().decode())
    return _lib


def last_error() -> str:
    return load().b200asr_last_error().decode()


def check(rc: int, what: str = ""):
    if rc != 0:
        raise RuntimeError(f"libb200asr {what} failed (code {rc}): {last_error()}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()
