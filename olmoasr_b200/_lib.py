"""ctypes binding of liboasr_b200.so (the C ABI declared in include/oasr_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, an exception is
raised.  Nothing in the product path computes on the CPU or through stock torch ops.
"""
from __future__ import annotations

import ctypes
import os
from pathlib import Path

import torch

# OASR_B200_LIB points at an alternative build of the same library (A/B measurements of kernel variants); it must
# export the same ABI -- there is still no non-CUDA fallback.
_LIB_PATH = Path(os.environ.get("OASR_B200_LIB") or Path(__file__).resolve().parent / "csrc" / "liboasr_b200.so")
_lib = None

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_float = ctypes.c_float


class OasrError(RuntimeError):
    pass


c_i32 = ctypes.c_int32
c_float_p = ctypes.c_void_p
DTYPE_BF16, DTYPE_F16, DTYPE_F32 = 0, 1, 2


class DecLinearArgs(ctypes.Structure):  # oasr_dec_linear_args (include/oasr_b200.h)
    _fields_ = [("x", c_void_p), ("ldx", c_i64), ("x_mode", c_i32), ("n_partials", c_i32), ("partial_stride", c_i64),
                ("ln_gamma", c_void_p), ("ln_beta", c_void_p), ("ln_eps", c_float), ("epi", c_i32),
                ("W", c_void_p), ("bias", c_void_p),
                ("out", c_void_p), ("ldo", c_i64), ("res", c_void_p), ("ldres", c_i64),
                ("k_cache", c_void_p), ("v_cache", c_void_p), ("cache_len", c_i64), ("pos_ptr", c_void_p),
                ("M", c_i32), ("N", c_i32), ("K", c_i32), ("dtype", c_i32)]


class DecAttnArgs(ctypes.Structure):  # oasr_dec_attn_args
    _fields_ = [("q", c_void_p), ("ldq", c_i64),
                ("k", c_void_p), ("v", c_void_p), ("kv_seq_stride", c_i64), ("kv_row_stride", c_i64),
                ("scores", c_void_p), ("scores_ld", c_i64),
                ("out_partial", c_void_p), ("ld_out", c_i64),
                ("pos_ptr", c_void_p), ("n_keys", c_i32),
                ("n_seq", c_i32), ("n_head", c_i32), ("n_splits", c_i32), ("scale", c_float), ("dtype", c_i32)]


class DecSampleArgs(ctypes.Structure):  # oasr_dec_sample_args
    _fields_ = [("logits", c_void_p), ("ld_logits", c_i64), ("tokens", c_void_p), ("ld_tokens", c_i64), ("pos_ptr", c_void_p),
                ("suppress", c_void_p), ("sum_logprobs", c_void_p), ("no_speech_prob", c_void_p), ("n_unfinished", c_void_p),
                ("done_flag", c_void_p), ("scratch", c_void_p), ("counters", c_void_p),
                ("n_seq", c_i32), ("n_vocab", c_i32), ("sample_begin", c_i32), ("sot_index", c_i32), ("suppress_blank", c_i32),
                ("blank", c_i32), ("eot", c_i32), ("no_speech", c_i32), ("n_slices", c_i32), ("reserved", c_i32)]


class DecSampleRulesArgs(ctypes.Structure):  # oasr_dec_sample_rules_args
    _fields_ = [("logits", c_void_p), ("ld_logits", c_i64), ("tokens", c_void_p), ("ld_tokens", c_i64), ("pos_ptr", c_void_p),
                ("suppress", c_void_p), ("sum_logprobs", c_void_p), ("no_speech_prob", c_void_p), ("n_unfinished", c_void_p),
                ("done_flag", c_void_p), ("scratch", c_void_p), ("counters", c_void_p), ("temperature", c_void_p),
                ("row_keys", c_void_p),
                ("n_seq", c_i32), ("n_vocab", c_i32), ("sample_begin", c_i32), ("sot_index", c_i32), ("suppress_blank", c_i32),
                ("blank", c_i32), ("eot", c_i32), ("no_speech", c_i32), ("n_slices", c_i32),
                ("timestamps", c_i32), ("timestamp_begin", c_i32), ("no_timestamps", c_i32), ("max_initial_timestamp", c_i32),
                ("reserved", c_i32)]


class DecBeamArgs(ctypes.Structure):  # oasr_dec_beam_args
    _fields_ = [("logits", c_void_p), ("ld_logits", c_i64), ("tokens", c_void_p), ("ld_tokens", c_i64), ("pos_ptr", c_void_p),
                ("suppress", c_void_p), ("sum_logprobs", c_void_p), ("no_speech_prob", c_void_p), ("n_unfinished", c_void_p),
                ("done_flag", c_void_p), ("scratch", c_void_p), ("src_rows", c_void_p),
                ("fin_tokens", c_void_p), ("ld_fin", c_i64), ("fin_scores", c_void_p), ("fin_len", c_void_p),
                ("fin_count", c_void_p), ("seq_len", c_void_p),
                ("n_clips", c_i32), ("beam", c_i32), ("max_candidates", c_i32), ("n_vocab", c_i32), ("n_slices", c_i32),
                ("n_ctx", c_i32), ("sample_begin", c_i32), ("sot_index", c_i32), ("suppress_blank", c_i32), ("blank", c_i32),
                ("eot", c_i32), ("no_speech", c_i32), ("timestamps", c_i32), ("timestamp_begin", c_i32),
                ("no_timestamps", c_i32), ("max_initial_timestamp", c_i32)]


# name -> argtypes (restype is always int unless listed in _RESTYPES)
_SIGNATURES = {
    "oasr_abi_version": [],
    "oasr_device_sm_count": [],
    "oasr_gemm_set_sm_budget": [c_int],
    "oasr_logmel": [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                    c_i64, c_i64, c_i64, c_i64, c_void_p],
    "oasr_layernorm_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_float, c_void_p],
    "oasr_layernorm_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                           c_i64, c_i64, c_void_p],
    "oasr_attention_fwd": [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p,
                           c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p, c_float, c_void_p],
    "oasr_attention_bwd": [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64,
                           c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64,
                           c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p, c_float, c_void_p],
    "oasr_ce_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_void_p],
    "oasr_ce_finalize": [c_void_p, c_void_p, c_void_p],
    "oasr_ce_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_void_p],
    "oasr_logits_to_f32": [c_void_p, c_void_p, c_i64, c_i64, c_i64, c_void_p],
    "oasr_embed_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_void_p],
    "oasr_embed_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_void_p],
    "oasr_cast_f32_to_bf16": [c_void_p, c_void_p, c_i64, c_void_p],
    "oasr_cast_conv_weight": [c_void_p, c_void_p, c_i64, c_i64, c_void_p],
    "oasr_unpermute_conv_wgrad": [c_void_p, c_void_p, c_i64, c_i64, c_int, c_void_p],
    "oasr_mask_to_kvlen": [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_void_p],
    "oasr_im2col_conv1": [c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_void_p],
    "oasr_im2col_conv2": [c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_void_p],
    "oasr_col2im_conv2_gelu_bwd": [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_void_p],
    "oasr_add_pos": [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_void_p],
    "oasr_gelu_bwd": [c_void_p, c_void_p, c_void_p, c_i64, c_void_p],
    "oasr_colsum_bf16": [c_void_p, c_void_p, c_i64, c_i64, c_i64, c_void_p],
    "oasr_optim_chunk_elems": [],
    "oasr_grad_sqnorm": [c_void_p, c_void_p, c_i64, c_float, c_void_p, c_void_p],
    "oasr_grad_sqnorm_flat": [c_void_p, c_i64, c_float, c_void_p, c_void_p],
    "oasr_optim_prepare": [c_void_p, c_void_p, c_void_p, c_float, c_float, c_float, c_float, c_void_p],
    "oasr_adamw_step": [c_void_p, c_void_p, c_i64, c_void_p, c_float, c_float, c_float, c_float, c_float, c_void_p],
    "oasr_adamw_flat": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_float, c_float, c_float,
                        c_float, c_float, c_void_p],
    "oasr_dec_embed": [c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_dec_linear": [ctypes.POINTER(DecLinearArgs), c_void_p],
    "oasr_dec_attention": [ctypes.POINTER(DecAttnArgs), c_void_p],
    "oasr_dec_sample": [ctypes.POINTER(DecSampleArgs), c_void_p],
    "oasr_dec_sample_rules": [ctypes.POINTER(DecSampleRulesArgs), c_void_p],
    "oasr_dec_attention_grouped": [ctypes.POINTER(DecAttnArgs), c_int, c_void_p],
    "oasr_dec_beam_candidates": [ctypes.POINTER(DecBeamArgs), c_void_p],
    "oasr_dec_beam_select": [ctypes.POINTER(DecBeamArgs), c_void_p],
    "oasr_dec_beam_reorder": [c_void_p, c_void_p, c_i64, c_i64, c_i64, c_void_p, c_void_p, c_i32, c_i32, c_i32, c_i32, c_int,
                              c_void_p],
    "oasr_convert": [c_void_p, c_int, c_void_p, c_int, c_i64, c_void_p],
    "oasr_gemm_bf16": [c_void_p, c_i64, c_int, c_void_p, c_i64, c_int, c_void_p, c_i64, c_void_p, c_void_p,
                       c_void_p, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_void_p],
    # 16-bit activation dtype (OASR_DTYPE_BF16 / OASR_DTYPE_F16) before the stream
    "oasr_gemm16": [c_void_p, c_i64, c_int, c_void_p, c_i64, c_int, c_void_p, c_i64, c_void_p, c_void_p,
                    c_void_p, c_i64, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_int, c_void_p],
    "oasr_layernorm_fwd16": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_float, c_int, c_void_p],
    "oasr_layernorm_bwd16": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_i64, c_i64, c_int, c_void_p],
    "oasr_attention_fwd16": [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p,
                             c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p, c_float, c_int, c_void_p],
    "oasr_attention_bwd16": [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64,
                             c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64,
                             c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p, c_float, c_int, c_void_p],
    "oasr_ce_fwd16": [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_ce_bwd16": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_logits_to_f32_16": [c_void_p, c_void_p, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_embed_fwd16": [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_embed_bwd16": [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_cast_conv_weight16": [c_void_p, c_void_p, c_i64, c_i64, c_int, c_void_p],
    "oasr_im2col_conv1_16": [c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_col2im_conv2_gelu_bwd16": [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_add_pos16": [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_gelu_bwd16": [c_void_p, c_void_p, c_void_p, c_i64, c_int, c_void_p],
    "oasr_colsum16": [c_void_p, c_void_p, c_i64, c_i64, c_i64, c_int, c_void_p],
    "oasr_adamw_flat16": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_float, c_float, c_float,
                          c_float, c_float, c_int, c_void_p],
    "oasr_optim_prepare_amp": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_float, c_float, c_void_p],
    # word-level timestamps: heads table of oasr_align_head {q, k, ldq, ldk}
    "oasr_align_cost": [c_void_p, c_i32, c_i32, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_i64, c_int, c_void_p],
    "oasr_dtw": [c_void_p, c_i64, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
}
_RESTYPES = {"oasr_last_error": ctypes.c_char_p}


def lib_path() -> Path:
    return _LIB_PATH


def lib():
    """Load (once) and return the ctypes handle.  Raises OasrError when the library is absent."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise OasrError(
                f"{_LIB_PATH} not found: build it with `python -m olmoasr_b200.build` "
                "(there is no CPU / eager fallback)"
            )
        h = ctypes.CDLL(str(_LIB_PATH), mode=ctypes.RTLD_GLOBAL)
        h.oasr_last_error.restype = ctypes.c_char_p
        h.oasr_last_error.argtypes = []
        for name, args in _SIGNATURES.items():
            fn = getattr(h, name)
            fn.argtypes = args
            fn.restype = _RESTYPES.get(name, c_int)
        _lib = h
    return _lib


def exported_symbols():
    """Names the header declares (used by the CPU-side ABI test)."""
    return ["oasr_last_error", *_SIGNATURES.keys()]


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().oasr_last_error()
        raise OasrError(f"{what or 'oasr call'} failed (rc={rc}): {msg.decode() if msg else ''}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
_cur_device = getattr(torch._C, "_cuda_getDevice", None)


def stream():
    """cudaStream_t of torch's current stream on the current device (the raw accessors avoid ~14 us of Stream-object
    construction per launch)."""
    if _raw_stream is not None and _cur_device is not None:
        return _raw_stream(_cur_device())
    return torch.cuda.current_stream().cuda_stream


# kernels launched per entry point (memsets not counted) -- bench.py reports the total as `gpu_launches`
_LAUNCHES_PER_CALL = {"oasr_logmel": 3, "oasr_attention_bwd": 3, "oasr_dec_attention": 2, "oasr_dec_sample": 2,
                      "oasr_dec_sample_rules": 2, "oasr_dec_attention_grouped": 2, "oasr_dec_beam_select": 2,
                      "oasr_ce_fwd": 2, "oasr_colsum_bf16": 2, "oasr_layernorm_bwd": 3, "oasr_grad_sqnorm": 2,
                      "oasr_grad_sqnorm_flat": 2, "oasr_attention_bwd16": 3, "oasr_ce_fwd16": 2, "oasr_colsum16": 2,
                      "oasr_layernorm_bwd16": 3, "oasr_align_cost": 2}
LAUNCH_COUNT = 0


def call(name: str, *args):
    global LAUNCH_COUNT
    fn = getattr(lib(), name)
    check(fn(*args), name)
    LAUNCH_COUNT += _LAUNCHES_PER_CALL.get(name, 1)
