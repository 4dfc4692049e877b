"""ctypes binding of libtaco_b200.so (include/taco_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, an
exception is raised.  Nothing here imports oracle/.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtaco_b200.so")

ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH = 0, 1, 2, 3
IMPL_TC, IMPL_SIMT, IMPL_TC3 = 0, 1, 2
EPI_NORMAL, EPI_HIGHWAY = 0, 1
DEC_INFER, DEC_TEACHER, DEC_SCHED = 0, 1, 2


class LinearDesc(C.Structure):
    _fields_ = [
        ("X", C.c_void_p), ("ldx", C.c_int64),
        ("B", C.c_int32), ("T", C.c_int32), ("C", C.c_int32),
        ("taps", C.c_int32), ("tap0", C.c_int32), ("N", C.c_int32),
        ("bank_K", C.c_int32), ("bank_cout", C.c_int32),
        ("W", C.c_void_p), ("Wp", C.c_void_p), ("ldwp", C.c_int64),
        ("Y", C.c_void_p), ("ldy", C.c_int64),
        ("bias", C.c_void_p), ("act", C.c_int32),
        ("scale", C.c_void_p), ("shift", C.c_void_p),
        ("keep", C.c_void_p), ("keep_scale", C.c_float),
        ("residual", C.c_void_p), ("ldr", C.c_int64),
        ("epilogue", C.c_int32),
        ("hx", C.c_void_p), ("ldhx", C.c_int64),
        ("pool", C.c_int32), ("impl", C.c_int32),
        ("bias_utt", C.c_void_p), ("ldbu", C.c_int64),
    ]


HIGHWAY_STACK_MAX = 4


class HighwayStackDesc(C.Structure):
    _fields_ = [
        ("X", C.c_void_p), ("ldx", C.c_int64), ("M", C.c_int32), ("C", C.c_int32),
        ("Wd_p", C.c_void_p), ("ldwd", C.c_int64), ("bd", C.c_void_p),
        ("L", C.c_int32),
        ("hw_p", C.c_void_p * HIGHWAY_STACK_MAX), ("ldhw", C.c_int64), ("hw_b", C.c_void_p * HIGHWAY_STACK_MAX),
        ("xp_p", C.c_void_p), ("ldxp", C.c_int64), ("xp_b", C.c_void_p),
        ("Y", C.c_void_p), ("ldy", C.c_int64),
        ("impl", C.c_int32),
    ]


class DecoderWeights(C.Structure):
    _fields_ = [
        ("pre_W1", C.c_void_p), ("pre_b1", C.c_void_p), ("pre_W2", C.c_void_p), ("pre_b2", C.c_void_p),
        ("in_W", C.c_void_p), ("in_b", C.c_void_p),
        ("gru_Wg", C.c_void_p * 3), ("gru_bg", C.c_void_p * 3), ("gru_Wc", C.c_void_p * 3), ("gru_bc", C.c_void_p * 3),
        ("out_W", C.c_void_p), ("out_b", C.c_void_p),
        ("att_Wq", C.c_void_p), ("att_v", C.c_void_p), ("att_Wa", C.c_void_p),
    ]


class DecoderArgs(C.Structure):
    _fields_ = [
        ("weights", C.POINTER(DecoderWeights)),
        ("packed", C.c_void_p), ("keys", C.c_void_p), ("values", C.c_void_p), ("text_length", C.c_void_p),
        ("mel", C.c_void_p), ("sample_mask", C.c_void_p), ("keep1", C.c_void_p), ("keep2", C.c_void_p),
        ("keep_scale", C.c_float), ("mode", C.c_int32),
        ("B", C.c_int32), ("Tx", C.c_int32), ("T", C.c_int32), ("r", C.c_int32),
        ("y", C.c_void_p), ("align", C.c_void_p), ("workspace", C.c_void_p), ("step_ns", C.c_void_p),
        ("h_save", C.c_void_p),
        ("row0", C.c_int32), ("row_stride", C.c_int32), ("max_ctas", C.c_int32),
        ("h0", C.c_void_p), ("att0", C.c_void_p),
        ("win_back", C.c_int32), ("win_ahead", C.c_int32), ("peak", C.c_void_p),
        ("stop_at", C.c_void_p), ("stop_hold", C.c_int32), ("end_step", C.c_void_p),
    ]


DECODER_STOP_LAG = 3      # TACO_DECODER_STOP_LAG (include/taco_b200.h)


class GemmDesc(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("lda", C.c_int64), ("B", C.c_void_p), ("ldb", C.c_int64), ("C", C.c_void_p), ("ldc", C.c_int64),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32), ("ta", C.c_int32), ("tb", C.c_int32), ("beta", C.c_float),
        ("shift", C.c_int32), ("period", C.c_int32), ("taps", C.c_int32), ("dshift", C.c_int32), ("kper", C.c_int32),
        ("b_tap_stride", C.c_int64), ("batch", C.c_int32),
        ("a_bstride", C.c_int64), ("b_bstride", C.c_int64), ("c_bstride", C.c_int64), ("bshift", C.c_int32),
    ]


class DecoderBwdArgs(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("T", C.c_int32), ("Tx", C.c_int32), ("r", C.c_int32), ("keep_scale", C.c_float),
        ("W_a", C.c_void_p), ("W_q", C.c_void_p), ("W_out", C.c_void_p), ("W_in", C.c_void_p), ("W1", C.c_void_p),
        ("W2", C.c_void_p), ("v", C.c_void_p),
        ("Wg", C.c_void_p * 3), ("Wc", C.c_void_p * 3),
        ("dy_ext", C.c_void_p),
        ("RU", C.c_void_p * 3), ("C", C.c_void_p * 3), ("H", C.c_void_p * 3),
        ("align", C.c_void_p), ("values", C.c_void_p), ("keys", C.c_void_p),
        ("PQ", C.c_void_p), ("PN1", C.c_void_p), ("PN2", C.c_void_p), ("sel", C.c_void_p),
        ("DATT", C.c_void_p), ("DY", C.c_void_p), ("DPQ", C.c_void_p), ("DSCORE", C.c_void_p),
        ("DCTX", C.c_void_p), ("DG", C.c_void_p * 3), ("DC", C.c_void_p * 3), ("DZ", C.c_void_p), ("DPN2", C.c_void_p),
        ("DPN1", C.c_void_p), ("DX", C.c_void_p), ("workspace", C.c_void_p), ("max_ctas", C.c_int32),
        ("H0", C.c_void_p * 3), ("DH0", C.c_void_p), ("dscore_add", C.c_void_p),
    ]


class TacoError(RuntimeError):
    pass


_lib = None

vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float

# every symbol include/taco_b200.h declares -> (restype, argtypes); tests check that the .so exports exactly these
SIGNATURES = {
    "taco_last_error": (C.c_char_p, []),
    "taco_version": (i32, []),
    "taco_device_info": (i32, [C.POINTER(C.c_int)] * 3),
    "taco_linear_fwd": (i32, [C.POINTER(LinearDesc), vp]),
    "taco_linear_route": (i32, [C.POINTER(LinearDesc)] + [C.POINTER(C.c_int)] * 5),
    "taco_pack_weight": (i32, [vp, i32, i32, i32, vp, i64, vp]),
    "taco_pack_weight_x3": (i32, [vp, i32, i32, i32, vp, vp, i64, vp]),
    "taco_highway_stack_fwd": (i32, [C.POINTER(HighwayStackDesc), vp]),
    "taco_maxpool_fwd": (i32, [vp, vp, i32, i32, i32, vp]),
    "taco_gather_rows": (i32, [vp, vp, i32, i32, i32, vp, f32, vp, vp]),
    "taco_mask_rows": (i32, [vp, vp, vp, i32, i32, i32, vp]),
    "taco_bigru_fwd": (i32, [vp] * 6 + [i32, i32, vp]),
    "taco_bigru_fwd_h0": (i32, [vp] * 8 + [i32, i32, vp]),
    "taco_decoder_packed_bytes": (C.c_size_t, [i32]),
    "taco_decoder_workspace_bytes": (C.c_size_t, [i32] * 4),
    "taco_decoder_trace_offset": (i64, []),
    "taco_decoder_pack": (i32, [C.POINTER(DecoderWeights), i32, vp, vp]),
    "taco_decoder_fwd": (i32, [C.POINTER(DecoderArgs), vp]),
    "taco_decoder_capacity": (i32, [C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "taco_l1_loss_fwd": (i32, [vp, vp, i64, vp, vp, vp]),
    "taco_l1_partial_count": (i32, []),
    "taco_launch_count": (C.c_ulonglong, []),
    # training path
    "taco_gemm": (i32, [C.POINTER(GemmDesc), vp]),
    "taco_set_gemm_impl": (i32, [i32]),
    "taco_conv_dw": (i32, [vp, i64, i64, vp, i64, vp, i64] + [C.c_int32] * 6 + [vp]),
    "taco_colsum": (i32, [vp, vp, i64, vp, i64, vp, i64, i32, i32, vp]),
    "taco_colsum_seg": (i32, [vp, i64, vp, i64, i32, i32, i32, vp]),
    "taco_bias_act": (i32, [vp, i64, i32, i32, vp, i32, vp]),
    "taco_mul_shift": (i32, [vp, i64, vp, i64, vp, i64, i32, i32, i32, i32, vp]),
    "taco_epi_bwd": (i32, [vp, i64, vp, i64, vp, i64, vp, i64, i32, i32, i32, vp, vp, f32, vp]),
    "taco_epi_fwd_keep": (i32, [vp, i64, vp, i32, i32, f32, vp]),
    "taco_bn_param_grad": (i32, [vp, vp, vp, vp, vp, vp, i32, vp]),
    "taco_maxpool_bwd": (i32, [vp, vp, vp, i32, i32, i32, vp]),
    "taco_highway_fwd": (i32, [vp, i64, vp, i64, vp, i64, i32, i32, vp]),
    "taco_highway_bwd": (i32, [vp, i64, vp, i64, vp, i64, vp, i64, vp, i64, i32, i32, vp]),
    "taco_l1_bwd": (i32, [vp, vp, vp, i64, f32, vp]),
    "taco_l1_bwd_ld": (i32, [vp, i64, vp, vp, i64, i64, f32, vp]),
    "taco_scatter_add_rows": (i32, [vp, vp, vp, i32, i32, i32, vp]),
    "taco_bigru_bwd": (i32, [vp] * 8 + [i32, i32, vp]),
    "taco_bigru_bwd_h0": (i32, [vp] * 11 + [i32, i32, vp]),
    "taco_dec_inputs": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "taco_decoder_bwd_workspace_bytes": (C.c_size_t, []),
    "taco_decoder_bwd": (i32, [C.POINTER(DecoderBwdArgs), vp]),
    "taco_attn_bwd_post": (i32, [vp, vp, vp, vp, vp, vp, i32, i32, i32, vp]),
    "taco_sumsq": (i32, [vp, i64, vp, vp, vp]),
    "taco_adam_step": (i32, [vp, vp, vp, vp, i64, f32, f32, f32, f32, f32, vp, vp]),
    # guided attention loss (opt-in training term)
    "taco_guided_attention": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, f32, f32, vp, vp]),
    "taco_guided_attention_partial_count": (i32, [i32, i32]),
    # spectrogram inversion (Griffin-Lim glue kernels)
    "taco_gl_init": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp]),
    "taco_gl_ola": (i32, [vp, vp, i32, i32, i32, i32, i32, vp]),
    "taco_gl_frame": (i32, [vp, vp, i32, i32, i32, i32, i32, vp]),
    "taco_gl_phase": (i32, [vp, vp, vp, i64, vp]),
    "taco_rfft2048": (i32, [vp, vp, i64, vp]),
    "taco_irfft2048": (i32, [vp, vp, i64, vp]),
    # end of speech and the packed Griffin-Lim kernels (synthesis tail trim)
    "taco_speech_frames": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, f32, vp]),
    "taco_gl_init_packed": (i32, [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, vp, vp, vp]),
    "taco_gl_ola_packed": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, vp]),
    "taco_gl_frame_packed": (i32, [vp, vp, vp, i32, i32, i32, i32, i32, vp]),
    # where speech starts and ends, and the join of synthesised pieces (long-form synthesis)
    "taco_speech_bounds": (i32, [vp, vp, i32, i32, i32, i32, vp, vp, f32, vp]),
    "taco_join_segments": (i32, [vp, i64, vp, vp, i32, i32, i32, vp]),
    # fast Griffin-Lim and de-emphasis (opt-in synthesis options)
    "taco_gl_phase_momentum": (i32, [vp, vp, vp, vp, f32, i64, vp]),
    "taco_de_emphasis": (i32, [vp, vp, i32, f32, vp]),
    # input data format
    "taco_normalize_f16": (i32, [vp, vp, vp, vp, i64, i32, vp]),
    # feature extraction (preprocessing)
    "taco_trim_bounds": (i32, [vp, vp, vp, i32, i32, i32, f32, vp]),
    "taco_feature_frames": (i32, [vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, f32, vp]),
    "taco_feature_spec": (i32, [vp, vp, i32, vp, vp, vp, vp, i32, i32, i32, i32, vp]),
    "taco_resample": (i32, [vp, vp, vp, vp, i32, vp, i32, i32, C.c_double, vp, i64, vp]),
    # training summaries
    "taco_histogram_workspace_bytes": (C.c_size_t, []),
    "taco_histogram": (i32, [vp, i64, vp, i32, vp, vp, vp, vp, vp]),
}
EXPORTS = list(SIGNATURES)


def declare(cdll, names=EXPORTS):
    """Give each named entry point of cdll (this library, or a build of the same sources) its SIGNATURES entry."""
    for name in names:
        fn = getattr(cdll, name)                  # a symbol that does not resolve raises AttributeError
        fn.restype, fn.argtypes = SIGNATURES[name]
    return cdll


def lib():
    """Load (once) and return the shared library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TacoError(
            f"{LIB_PATH} not found: the CUDA extension has not been built (run `python -m tacotron_b200.build` "
            "or __graft_entry__.build()). There is no CPU fallback.")
    _lib = declare(C.CDLL(LIB_PATH))              # every declared symbol must resolve
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().taco_last_error().decode("utf-8", "replace")
        raise TacoError(f"{what} failed (rc={rc}): {msg}")


def linear_route(d):
    """(bn, stages, mode, direct, tile_stride) of the launch taco_linear_fwd makes for LinearDesc d (host only)."""
    out = [C.c_int() for _ in range(5)]
    check(lib().taco_linear_route(C.byref(d), *[C.byref(v) for v in out]), "taco_linear_route")
    return tuple(v.value for v in out)


def ptr(t):
    """Device pointer of a torch tensor (or None -> NULL)."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def current_stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
