"""ctypes binding of libmt3b200.so (the C ABI declared in include/mt3_b200.h).

Fails loudly: a missing library is an ImportError-like RuntimeError, a non-zero status
from any entry point raises Mt3Error with mt3_last_error().  Nothing here falls back
to a CPU path.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libmt3b200.so")

MT3_OK = 0
GEMM_FP32_SIMT, GEMM_TF32X3, GEMM_TF32 = 0, 1, 2
KV_F32, KV_F16, KV_P24 = 0, 1, 2
GEN_STOP_AT_EOS, GEN_USE_GRAPH, GEN_BEAM1, GEN_SAMPLE = 1, 2, 4, 8
ABI_VERSION = 2
K_DEC_SELF_ATTN, K_DEC_CROSS_ATTN, K_DEC_QKV_GEMM, K_ENC_QKV_GEMM, K_ENC_ATTN = 0, 1, 2, 3, 4

EXPORTS = [
    "mt3_abi_version", "mt3_last_error", "mt3_kernel_launch_count",
    "mt3_frontend_create", "mt3_frontend_destroy", "mt3_frontend_num_frames", "mt3_logmel_f32",
    "mt3_model_num_params", "mt3_model_param_offset", "mt3_model_create", "mt3_model_destroy",
    "mt3_workspace_bytes", "mt3_model_set_workspace", "mt3_encode", "mt3_cross_kv", "mt3_decode_step",
    "mt3_generate", "mt3_generate_scored", "mt3_vocab_decode", "mt3_dot_product_attention_f32", "mt3_debug_launch", "mt3_debug_trace_step",
    "mt3_teacher_forced_workspace_bytes", "mt3_decode_teacher_forced", "mt3_generate_prompted", "mt3_generate_sampled",
    "mt3_generate_biased",
]


class Mt3Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"mt3_b200 error {code}: {msg}")
        self.code = code


class FrontendConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("hop_width", C.c_int32), ("fft_size", C.c_int32),
                ("num_mel_bins", C.c_int32), ("log_eps", C.c_float)]


class ModelConfig(C.Structure):
    _fields_ = [("vocab_size", C.c_int32), ("emb_dim", C.c_int32), ("num_heads", C.c_int32),
                ("head_dim", C.c_int32), ("num_encoder_layers", C.c_int32), ("num_decoder_layers", C.c_int32),
                ("mlp_dim", C.c_int32), ("input_depth", C.c_int32), ("max_batch", C.c_int32),
                ("max_input_length", C.c_int32), ("max_decode_length", C.c_int32), ("gemm_mode", C.c_int32),
                ("kv_cache_format", C.c_int32)]


class SampleParams(C.Structure):
    _fields_ = [("temperature", C.c_float), ("topk", C.c_int32), ("topp", C.c_float), ("key", C.c_uint32 * 2),
                ("row0", C.c_uint32), ("rescale_log_probs", C.c_int32)]


_lib = None


def load() -> C.CDLL:
    """Loads the library (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -m mt3_b200.build` (nvcc, sm_90a). "
            "mt3_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, f32p, i32p = C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p
    lib.mt3_abi_version.restype = C.c_int
    lib.mt3_last_error.restype = C.c_char_p
    lib.mt3_kernel_launch_count.restype = C.c_uint64
    lib.mt3_frontend_create.argtypes = [C.POINTER(FrontendConfig), vp, C.POINTER(vp)]
    lib.mt3_frontend_destroy.argtypes = [vp]
    lib.mt3_frontend_num_frames.argtypes = [vp, i64]
    lib.mt3_logmel_f32.argtypes = [vp, f32p, i64, i32, i32, i32p, f32p, vp]
    lib.mt3_model_num_params.argtypes = [C.POINTER(ModelConfig)]
    lib.mt3_model_num_params.restype = i64
    lib.mt3_model_param_offset.argtypes = [C.POINTER(ModelConfig), C.c_char_p, C.POINTER(i64)]
    lib.mt3_model_param_offset.restype = i64
    lib.mt3_model_create.argtypes = [C.POINTER(ModelConfig), f32p, C.POINTER(vp), vp]
    lib.mt3_model_destroy.argtypes = [vp]
    lib.mt3_workspace_bytes.argtypes = [vp, i32, i32]
    lib.mt3_workspace_bytes.restype = i64
    lib.mt3_model_set_workspace.argtypes = [vp, vp, i64, i32, i32]
    lib.mt3_encode.argtypes = [vp, f32p, f32p, vp]
    lib.mt3_cross_kv.argtypes = [vp, f32p, vp]
    lib.mt3_decode_step.argtypes = [vp, i32p, f32p, i32p, vp]
    lib.mt3_generate.argtypes = [vp, f32p, i32, i32, i32p, C.POINTER(i32), vp]
    lib.mt3_generate_scored.argtypes = [vp, f32p, i32, i32, i32p, f32p, f32p, C.POINTER(i32), vp]
    lib.mt3_generate_prompted.argtypes = [vp, f32p, i32, i32, i32p, i32, i32p, f32p, f32p, C.POINTER(i32), vp, i64, vp]
    lib.mt3_generate_sampled.argtypes = [vp, f32p, i32, i32, i32p, i32, i32p, f32p, f32p, C.POINTER(i32), vp, i64,
                                         C.POINTER(SampleParams), vp]
    lib.mt3_generate_biased.argtypes = [vp, f32p, i32, i32, i32p, i32, i32p, f32p, f32p, C.POINTER(i32), vp, i64,
                                        C.POINTER(SampleParams), f32p, i64, vp]
    lib.mt3_vocab_decode.argtypes = [i32p, i32, i32, i32, i32p, vp]
    lib.mt3_dot_product_attention_f32.argtypes = [f32p, f32p, f32p, f32p, i32, i32, i32, i32, i32, f32p, vp]
    lib.mt3_debug_launch.argtypes = [vp, i32, i32, i32, vp]
    lib.mt3_teacher_forced_workspace_bytes.argtypes = [vp, i32, i32, i32]
    lib.mt3_teacher_forced_workspace_bytes.restype = i64
    lib.mt3_decode_teacher_forced.argtypes = [vp, f32p, i32, i32, i32p, i32p, i32p, i32, f32p, f32p, vp, i64, vp]
    lib.mt3_debug_trace_step.argtypes = [vp, i32, vp, i32, C.c_char_p, i32, C.POINTER(C.c_int32), vp]
    for name in EXPORTS:
        getattr(lib, name)  # AttributeError here = header/library mismatch
    if lib.mt3_abi_version() != ABI_VERSION:
        raise RuntimeError(f"{LIB_PATH} has ABI version {lib.mt3_abi_version()}, this package binds version {ABI_VERSION}: "
                           "rebuild with `python -m mt3_b200.build --force`")
    _lib = lib
    return lib


def check(status: int) -> None:
    if status != MT3_OK:
        raise Mt3Error(status, load().mt3_last_error().decode("utf-8", "replace"))


def launch_count() -> int:
    return int(load().mt3_kernel_launch_count())
