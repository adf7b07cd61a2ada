"""ctypes binding of libpcm_b200.so (the C ABI declared in include/pcm_b200.h).

The product path has no CPU fallback: if the shared library is missing the import of any op
fails loudly with instructions to run ``python -c "import __graft_entry__ as g; g.build()"``.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# PCM_B200_LIB: alternative build of the same C ABI (kernel experiments); default = the in-tree library
LIB_PATH = os.environ.get("PCM_B200_LIB") or os.path.join(_HERE, "lib", "libpcm_b200.so")

MAX_ASRC, MAX_BSRC, MAX_PROG = 6, 4, 24
SUMSQ_WS_DOUBLES = 1024   # PCM_SUMSQ_WS_DOUBLES


class ASrc(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("C", C.c_int32), ("W", C.c_int32), ("H", C.c_int32),
                ("B", C.c_int32), ("sW", C.c_int64), ("sH", C.c_int64), ("sB", C.c_int64)]


class BSrc(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("K", C.c_int32), ("N", C.c_int32), ("ld", C.c_int64), ("kblocked", C.c_int32)]


class KEntry(C.Structure):
    _fields_ = [("a_src", C.c_int32), ("b_src", C.c_int32), ("dw", C.c_int32), ("dh", C.c_int32),
                ("nchunks", C.c_int32), ("a_c0", C.c_int32), ("b_k0", C.c_int32), ("n_lo", C.c_uint16), ("n_hi", C.c_uint16)]


class GemmDesc(C.Structure):
    _fields_ = [
        ("a", ASrc * MAX_ASRC), ("b", BSrc * MAX_BSRC), ("prog", KEntry * MAX_PROG),
        ("num_a", C.c_int32), ("num_b", C.c_int32), ("num_prog", C.c_int32),
        ("lin", C.c_int32), ("M", C.c_int32), ("N", C.c_int32),
        ("geoW", C.c_int32), ("geoH", C.c_int32), ("block_n", C.c_int32),
        ("out", C.c_void_p), ("bias", C.c_void_p), ("rowvec", C.c_void_p), ("residual", C.c_void_p),
        ("osW", C.c_int64), ("osH", C.c_int64), ("osB", C.c_int64), ("rowvec_ld", C.c_int64),
        ("epiW", C.c_int32), ("epiHW", C.c_int32), ("out_fp32", C.c_int32), ("round_bf16", C.c_int32),
        ("alpha", C.c_float), ("act", C.c_int32), ("ksplit", C.c_int32), ("splitk_ws", C.c_void_p),
        ("dep_a_src1", C.c_int32),
    ]


class WgradDesc(C.Structure):
    _fields_ = [
        ("p", ASrc), ("q", ASrc), ("q_c0", C.c_int32), ("lin", C.c_int32), ("M", C.c_int32),
        ("geoW", C.c_int32), ("geoH", C.c_int32), ("num_taps", C.c_int32),
        ("dw", C.c_int32 * 9), ("dh", C.c_int32 * 9), ("tap_off", C.c_int64 * 9),
        ("out", C.c_void_p), ("os_row", C.c_int64), ("os_col", C.c_int64),
        ("ksplit", C.c_int32), ("alpha", C.c_float), ("sem", C.c_void_p),
    ]


_lib = None


def lib():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: the pcm_b200 CUDA extension is not built. "
                "Run `python -c \"import __graft_entry__ as g; g.build()\"` (needs nvcc). "
                "There is no CPU fallback for the product path.")
        _lib = C.CDLL(LIB_PATH)
        _lib.pcm_last_error.restype = C.c_char_p
        for name in EXPORTS:
            fn = getattr(_lib, name)
            if name == "pcm_groupnorm_ws_bytes":
                fn.restype = C.c_int64
            elif name not in ("pcm_last_error",):
                fn.restype = C.c_int
            if name in ARGTYPES:
                fn.argtypes = ARGTYPES[name]
    return _lib


# every symbol include/pcm_b200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "pcm_last_error",
    "pcm_version",
    "pcm_num_sms",
    "pcm_gemm",
    "pcm_wgrad",
    "pcm_groupnorm_ws_bytes",
    "pcm_groupnorm_fwd",
    "pcm_groupnorm_fwd_part",
    "pcm_groupnorm_bwd",
    "pcm_layernorm_fwd",
    "pcm_layernorm_bwd",
    "pcm_attn_fwd",
    "pcm_attn_bwd",
    "pcm_geglu_fwd",
    "pcm_geglu_bwd",
    "pcm_upsample2x_fwd",
    "pcm_upsample2x_bwd",
    "pcm_conv3x3_c4",
    "pcm_timestep_embed",
    "pcm_colsum",
    "pcm_add_bf16",
    "pcm_cast_f32_bf16",
    "pcm_prepare",
    "pcm_add_noise",
    "pcm_teacher_step",
    "pcm_teacher_substep",
    "pcm_loss",
    "pcm_noise_travel",
    "pcm_axpby_f64",
    "pcm_fm_step",
    "pcm_grad_sumsq",
    "pcm_adamw_clip",
    "pcm_ema_update",
    "pcm_lora_refresh",
    "pcm_lora_fuse",
    "pcm_sample_step",
]


P, I, L64, F, D = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double
ARGTYPES = {
    "pcm_gemm": [P, P],
    "pcm_wgrad": [P, P],
    "pcm_groupnorm_ws_bytes": [I, I, I, I],
    "pcm_groupnorm_fwd": [P, P, I, I, I, I, I, P, P, F, I, P, P, P, L64, P],
    "pcm_groupnorm_fwd_part": [P, P, I, I, I, I, I, I, P, P, F, I, P, P, P, L64, P],
    "pcm_groupnorm_bwd": [P, P, P, I, I, I, I, I, P, P, F, I, P, P, P, P, P, P, P, L64, P],
    "pcm_layernorm_fwd": [P, I, I, P, P, F, P, P, P],
    "pcm_layernorm_bwd": [P, P, I, I, P, P, P, P, P],
    "pcm_attn_fwd": [P, P, P, P, P, I, I, I, I, I, L64, L64, L64, L64, F, P],
    "pcm_attn_bwd": [P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, L64, L64, L64, L64, F, P],
    "pcm_geglu_fwd": [P, L64, I, P, P],
    "pcm_geglu_bwd": [P, P, L64, I, P, P],
    "pcm_upsample2x_fwd": [P, I, I, I, I, P, P],
    "pcm_upsample2x_bwd": [P, I, I, I, I, P, P],
    "pcm_conv3x3_c4": [P, I, I, I, I, P, P, I, I, P, P],
    "pcm_timestep_embed": [P, I, I, P, P],
    "pcm_colsum": [P, I, I, I, P, P],
    "pcm_add_bf16": [P, P, L64, P, P],
    "pcm_cast_f32_bf16": [P, L64, P, P],
    "pcm_prepare": [P, I, I, P, I, P, P, I, I, P, P, P, P, P],
    "pcm_add_noise": [P, P, P, L64, I, I, P, P],
    "pcm_teacher_step": [P, P, P, P, L64, I, I, P, P],
    "pcm_teacher_substep": [P, P, P, P, P, P, P, L64, I, I, P, P],
    "pcm_loss": [P, P, P, P, P, L64, I, I, F, I, P, P, P, P, P],
    "pcm_noise_travel": [P, P, P, P, P, L64, I, P, P],
    "pcm_axpby_f64": [P, P, P, P, L64, I, P, P],
    "pcm_fm_step": [P, P, P, P, P, L64, I, I, P, P],
    "pcm_grad_sumsq": [P, L64, P, P],
    "pcm_adamw_clip": [P, P, P, P, L64, P, F, F, F, F, F, F, P, I, P],
    "pcm_ema_update": [P, P, L64, F, P],
    "pcm_lora_refresh": [P, P, I, L64, F, P, P],
    "pcm_lora_fuse": [P, P, I, L64, F, P],
    "pcm_sample_step": [P, P, P, P, L64, I, I, P, D, D, D, D, I, P],
}


class PcmError(RuntimeError):
    pass


def check(rc, what=""):
    if rc != 0:
        raise PcmError(f"{what} failed ({rc}): {lib().pcm_last_error().decode()}")
