"""ctypes binding of liblatte_b200.so (the C ABI in include/latte_b200.h).

There is no fallback: if the library is missing it is built with nvcc; if that fails, importing
raises.  Nothing here touches torch — the wrappers above pass raw device pointers.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

ABI_VERSION = 7
GEMM_SK_FLAGS = 1024   # B200_GEMM_SK_FLAGS: u64 words of the stream-K flag buffer
OK = 0
FP16, BF16 = 0, 1
EPI_BIAS, EPI_BIAS_GELU, EPI_GATE_RESIDUAL, EPI_BIAS_ADD16, EPI_BIAS_MUL16, EPI_BIAS_GELU_BOTH = 0, 1, 2, 3, 4, 5
VAE_CONV3X3, VAE_CONV_T3, VAE_CONV_DOWN2 = 0, 1, 2
ERR_NAMES = {-1: "SHAPE", -2: "DTYPE", -3: "ALIGN", -4: "ARCH", -5: "WORKSPACE", -6: "CUDA", -7: "UNSUPPORTED"}


class LatteShape(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "depth", "hidden", "heads", "mlp_hidden", "patch", "in_channels", "out_channels", "input_size",
        "frames", "num_embed", "dtype", "wide_patch")]


WEIGHT_FIELDS = (
    "patch_w", "patch_b", "pos_embed", "temp_embed", "t_w0", "t_b0", "t_w2", "t_b2", "y_table",
    "ada_w16", "ada_b", "qkv_w16", "qkv_b", "proj_w16", "proj_b", "fc1_w16", "fc1_b", "fc2_w16", "fc2_b",
    "final_w", "final_b", "final_w16", "qkv_w8", "qkv_ws", "fc1_w8", "fc1_ws")


class LatteWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in WEIGHT_FIELDS]


class T2VShape(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "layers", "hidden", "heads", "mlp_hidden", "patch", "in_channels", "out_channels", "input_size", "frames",
        "caption_channels", "dtype")]


T2V_WEIGHT_FIELDS = (
    "patch_w", "patch_b", "pos_embed", "temp_embed", "t_w0", "t_b0", "t_w2", "t_b2", "ada_w16", "ada_b",
    "cap_w1_16", "cap_b1", "cap_w2_16", "cap_b2", "tables", "final_table",
    "s_qkv_w16", "s_qkv_b", "s_out_w16", "s_out_b", "c_q_w16", "c_q_b", "c_kv_w16", "c_kv_b", "c_out_w16", "c_out_b",
    "s_fc1_w16", "s_fc1_b", "s_fc2_w16", "s_fc2_b",
    "t_qkv_w16", "t_qkv_b", "t_out_w16", "t_out_b", "t_fc1_w16", "t_fc1_b", "t_fc2_w16", "t_fc2_b", "final_w", "final_b",
    "final_w16", "s_qkv_w8", "s_qkv_ws", "s_fc1_w8", "s_fc1_ws", "t_qkv_w8", "t_qkv_ws", "t_fc1_w8", "t_fc1_ws")


class T2VWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in T2V_WEIGHT_FIELDS]


class T5Shape(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("layers", "d_model", "heads", "d_ff", "vocab", "dtype")] + [("eps", C.c_float)]


T5_WEIGHT_FIELDS = ("embed16", "qkv_w16", "o_w16", "ln0_w", "wi0_w16", "wi1_w16", "wo_w16", "ln1_w", "final_w")


class T5Weights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in T5_WEIGHT_FIELDS]


class VaeResnet(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("gn1_g", "gn1_b", "conv1_w16", "conv1_b", "gn2_g", "gn2_b", "conv2_w16", "conv2_b",
                                          "short_w16", "short_b")] + [("cin", C.c_int32), ("cout", C.c_int32)] + \
               [(n, C.c_void_p) for n in ("t_gn1_g", "t_gn1_b", "t_conv1_w16", "t_conv1_b", "t_gn2_g", "t_gn2_b", "t_conv2_w16", "t_conv2_b")]


class VaeDecoder(C.Structure):
    _fields_ = [("latent_channels", C.c_int32), ("layers_per_block", C.c_int32), ("n_up", C.c_int32), ("up_channels", C.c_int32 * 4),
                ("groups", C.c_int32), ("dtype", C.c_int32), ("eps", C.c_float),
                ("pq_w", C.c_void_p), ("pq_b", C.c_void_p), ("conv_in_w", C.c_void_p), ("conv_in_b", C.c_void_p),
                ("mid", VaeResnet * 2),
                ("attn_gn_g", C.c_void_p), ("attn_gn_b", C.c_void_p), ("attn_q_w16", C.c_void_p), ("attn_q_b", C.c_void_p),
                ("attn_k_w16", C.c_void_p), ("attn_k_b", C.c_void_p), ("attn_v_w16", C.c_void_p), ("attn_o_w16", C.c_void_p),
                ("attn_o_b", C.c_void_p),
                ("up", VaeResnet * 12), ("ups_w16", C.c_void_p * 3), ("ups_b", C.c_void_p * 3),
                ("norm_out_g", C.c_void_p), ("norm_out_b", C.c_void_p), ("conv_out_w16", C.c_void_p), ("conv_out_b", C.c_void_p),
                ("out_channels", C.c_int32), ("temporal_eps", C.c_float), ("time_conv_w", C.c_void_p), ("time_conv_b", C.c_void_p)]


class VaeEncoder(C.Structure):
    _fields_ = [("in_channels", C.c_int32), ("n_down", C.c_int32), ("down_channels", C.c_int32 * 4), ("groups", C.c_int32),
                ("dtype", C.c_int32), ("eps", C.c_float), ("latent_channels", C.c_int32),
                ("conv_in_w", C.c_void_p), ("conv_in_b", C.c_void_p),
                ("down", VaeResnet * 8), ("down_w16", C.c_void_p * 3), ("down_b", C.c_void_p * 3),
                ("mid", VaeResnet * 2),
                ("attn_gn_g", C.c_void_p), ("attn_gn_b", C.c_void_p), ("attn_q_w16", C.c_void_p), ("attn_q_b", C.c_void_p),
                ("attn_k_w16", C.c_void_p), ("attn_k_b", C.c_void_p), ("attn_v_w16", C.c_void_p), ("attn_o_w16", C.c_void_p),
                ("attn_o_b", C.c_void_p),
                ("norm_out_g", C.c_void_p), ("norm_out_b", C.c_void_p), ("conv_out_w16", C.c_void_p), ("conv_out_b", C.c_void_p),
                ("quant_w", C.c_void_p), ("quant_b", C.c_void_p)]


class SamplerTables(C.Structure):
    _fields_ = [("num_timesteps", C.c_int)] + [(n, C.c_void_p) for n in (
        "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_mean_coef1", "posterior_mean_coef2",
        "posterior_log_variance_clipped", "log_betas", "ddim_sqrt_alpha_prev", "ddim_sigma", "ddim_dir")]


EXPORTS = {
    "b200_last_error": (C.c_char_p, []),
    "b200_abi_version": (C.c_int, []),
    "b200_latte_workspace_bytes": (C.c_size_t, [C.POINTER(LatteShape), C.c_int]),
    "b200_latte_forward": (C.c_int, [C.POINTER(LatteShape), C.POINTER(LatteWeights), C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_size_t,
                                     C.c_void_p]),
    "b200_latte_conditioning_bytes": (C.c_size_t, [C.POINTER(LatteShape), C.c_int]),
    "b200_latte_conditioning_workspace_bytes": (C.c_size_t, [C.POINTER(LatteShape), C.c_int]),
    "b200_latte_conditioning": (C.c_int, [C.POINTER(LatteShape), C.POINTER(LatteWeights), C.c_void_p, C.c_void_p, C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_latte_forward_conditioned": (C.c_int, [C.POINTER(LatteShape), C.POINTER(LatteWeights), C.c_void_p, C.c_void_p,
                                                 C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_size_t,
                                                 C.c_void_p]),
    "b200_linear": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                 C.c_int, C.c_void_p]),
    "b200_ln_modulate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int,
                                   C.c_int, C.c_int, C.c_void_p]),
    # FP8 (e4m3) sampling path
    "b200_quantize_rows_e4m3": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_ln_modulate_e4m3": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_int, C.c_void_p]),
    "b200_linear_e4m3": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_int, C.c_void_p, C.c_void_p]),
    "b200_t2v_workspace_bytes": (C.c_size_t, [C.POINTER(T2VShape), C.c_int, C.c_int]),
    "b200_t2v_forward": (C.c_int, [C.POINTER(T2VShape), C.POINTER(T2VWeights), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_cross_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_frames_to_uint8": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200_t5_workspace_bytes": (C.c_size_t, [C.POINTER(T5Shape), C.c_int]),
    "b200_t5_encode": (C.c_int, [C.POINTER(T5Shape), C.POINTER(T5Weights), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_vae_workspace_bytes": (C.c_size_t, [C.POINTER(VaeDecoder), C.c_int, C.c_int, C.c_int]),
    "b200_vae_decode": (C.c_int, [C.POINTER(VaeDecoder), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t,
                                  C.c_void_p]),
    "b200_vae_encode_workspace_bytes": (C.c_size_t, [C.POINTER(VaeEncoder), C.c_int, C.c_int, C.c_int]),
    "b200_vae_encode": (C.c_int, [C.POINTER(VaeEncoder), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t,
                                  C.c_void_p]),
    "b200_vae_decode_temporal": (C.c_int, [C.POINTER(VaeDecoder), C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                           C.c_size_t, C.c_void_p]),
    "b200_vae_conv": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_group_norm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_float, C.c_int, C.c_int, C.c_void_p]),
    "b200_vae_mid_attention_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200_vae_mid_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                         C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "b200_sampler_step": (C.c_int, [C.POINTER(SamplerTables), C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_training_loss": (C.c_int, [C.POINTER(SamplerTables), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                     C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_wgrad_schedule": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                      C.POINTER(C.c_int32), C.c_int]),
    "b200_gemm_schedule": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                     C.POINTER(C.c_int), C.POINTER(C.c_int32), C.c_int]),
    # training-step passes (csrc/train.cu)
    "b200_wgrad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "b200_dgrad": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_linear_gelu_both": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "b200_transpose16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "b200_multi_cast": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_void_p]),
    "b200_multi_tensor": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "b200_cast16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]),
    "b200_gate_residual": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                     C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_gelu_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_gate_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_int64,
                                C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_colsum": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "b200_ln_modulate_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_int64, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_attention_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_cross_attention_bwd_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "b200_cross_attention_bwd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                           C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                           C.c_size_t, C.c_void_p]),
    "b200_ada_outer": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_ada_dsc": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "b200_profile_enable": (None, [C.c_int]),
    "b200_profile_collect": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_int]),
}

_lib = None


def lib_path() -> str:
    return _build.LIB


def load(rebuild_if_stale: bool = True):
    """Load (building first if needed) and type the library.  Raises on any failure."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not os.path.exists(path) or (rebuild_if_stale and os.environ.get("LATTE_B200_NO_BUILD") != "1"):
        try:
            _build.build_library()
        except Exception as e:  # a prebuilt .so that travelled to a box without nvcc is still usable
            if not os.path.exists(path):
                raise RuntimeError(f"liblatte_b200.so is missing and could not be built: {e}") from e
    lib = C.CDLL(path)
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    v = lib.b200_abi_version()
    if v != ABI_VERSION:
        raise RuntimeError(f"liblatte_b200.so ABI version {v} != expected {ABI_VERSION}; rebuild")
    _lib = lib
    return lib


_profiling = False


def profile_enable(on: bool) -> None:
    """bench.py's roofline hook (b200_profile_enable): CUDA events around every launch -- incompatible with graph replay,
    so the modules launch eagerly while it is on."""
    global _profiling
    load().b200_profile_enable(int(bool(on)))
    _profiling = bool(on)


def profiling_enabled() -> bool:
    return _profiling


def last_error() -> str:
    return load().b200_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != OK:
        raise RuntimeError(f"{what} failed: B200_ERR_{ERR_NAMES.get(rc, rc)}: {last_error()}")
