"""ctypes binding of libuav_b200.so (the C ABI declared in include/uav_b200.h and include/uav_b200_int8.h).

There is deliberately NO fallback: if the shared object is missing or a call fails, a
RuntimeError is raised (SURVEY.md §8b "Errors": non-zero status -> Python raises).
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libuav_b200.so"
_lib = None


class UavError(RuntimeError):
    pass


def require_cuda(t, who: str):
    """every public entry of the package refuses non-CUDA tensors: there is no CPU path.  (A single choke point so that the
    CPU test-suite can exercise the host logic against emulated kernels — tests/emu_ops.py — by stubbing exactly this.)"""
    if not t.is_cuda:
        raise UavError(f"{who}: CUDA tensors required — uav_b200 has no CPU path")


class Epilogue(C.Structure):
    """uav_epilogue_t"""
    _fields_ = [
        ("bias", C.c_void_p),
        ("rowvec", C.c_void_p),
        ("rows_per_vec", C.c_int64),
        ("ld_rowvec", C.c_int64),
        ("residual", C.c_void_p),
        ("ld_res", C.c_int64),
        ("act", C.c_int),
        ("out_dtype", C.c_int),
        ("ld_out", C.c_int64),
        ("out_scale", C.c_float),
        ("gn_partial", C.c_void_p),
        ("gn_blocks", C.c_int64),
    ]


class GnSource(C.Structure):
    """uav_gn_source_t"""
    _fields_ = [("partial", C.c_void_p), ("blocks", C.c_int64), ("C", C.c_int64), ("slabs", C.c_int64),
                ("x", C.c_void_p), ("ld", C.c_int64), ("slab_stride", C.c_int64)]


class CfgStep(C.Structure):
    """uav_cfg_step_t"""
    _fields_ = [("guidance_scale", C.c_float), ("pred_type", C.c_int), ("sqrt_alpha", C.c_float), ("sqrt_beta", C.c_float),
                ("clip", C.c_int), ("clip_range", C.c_float), ("sample", C.c_void_p), ("noise_pred", C.c_void_p),
                ("pred_original_sample", C.c_void_p)]


I64, I32, P, F32 = C.c_int64, C.c_int, C.c_void_p, C.c_float
EP = C.POINTER(Epilogue)

# name -> argtypes (restype is int status unless listed in _SPECIAL)
_PROTOS = {
    "uav_linear": [P, I64, I64, I64, P, I64, P, EP, P],
    "uav_conv2d": [P, I64, I64, I64, I64, I64, P, I64, I32, I32, I32, P, EP, P],
    "uav_conv_temporal": [P, I64, I64, I64, I64, I64, P, I64, I32, P, EP, P],
    "uav_conv3d": [P, I64, I64, I64, I64, I64, I64, P, I64, P, EP, P],
    "uav_upsample2x_conv3x3": [P, I64, I64, I64, I64, I64, P, I64, P, EP, P],
    "uav_groupnorm_silu": [P, I64, I64, I64, I64, I32, P, P, F32, I32, P, I64, P, C.c_size_t, P],
    "uav_groupnorm_silu_from_partials": [P, I64, I64, I64, I64, I32, P, P, F32, I32, P, I64, C.POINTER(GnSource), I32, P,
                                         C.c_size_t, P],
    "uav_groupnorm_affine": [P, I64, I64, I64, I64, I32, P, P, F32, C.POINTER(GnSource), I32, P, P, C.c_size_t, P],
    "uav_conv_out_fused": [P, I64, I64, I64, I64, I64, I64, P, P, P, I64, P, I32, P],
    "uav_conv_out_cfg_step": [P, I64, I64, I64, I64, I64, P, P, P, I64, C.POINTER(CfgStep), P],
    "uav_layernorm": [P, I64, I64, I64, P, P, F32, P, I64, P],
    "uav_attention": [P, P, P, P, I64, I32, I32, I64, I64, I64, I64, I64, I64, I64, F32, P],
    "uav_temporal_attention": [P, P, P, P, I64, I64, I64, I32, I32, I64, I64, I64, I64, F32, P, P, P],
    "uav_copy_channels": [P, I64, P, I64, I64, I64, P],
    "uav_upsample_nearest": [P, I64, I64, I64, I64, I64, P, I64, I64, I64, P],
    "uav_planar_to_channels_last": [P, I32, I64, I64, I64, P, I64, I64, F32, P],
    "uav_channels_last_to_planar": [P, I32, I64, I64, I64, I64, P, I32, I32, P],
    "uav_silu": [P, P, I64, P],
    "uav_sft_fuse": [P, P, P, F32, F32, P, I64, P],
    "uav_timestep_embedding": [P, I64, I64, I32, F32, P, P],
    "uav_cfg_combine": [P, P, I64, F32, I32, P],
    "uav_window_blend": [P, I64, P, I64, I64, C.c_uint32, I64, I64, I32, P],
    "uav_ddim_step_v0": [P, P, P, I64, I32, F32, F32, I32, F32, I32, P],
    "uav_ddim_step_vt": [P, P, P, P, I64, I32, F32, F32, F32, F32, I32, F32, F32, P, I32, P],
    "uav_add_noise": [P, P, P, I64, F32, F32, I32, P],
    "uav_propagate_step": [P, P, P, P, P, I64, I64, I64, I64, I64, I64, I64, I64, I32, I32, F32, F32, F32, I32, P],
    "uav_flow_resize_area": [P, P, I64, I64, I64, I64, I64, I64, I64, F32, I32, P],
    "uav_conv2d_taps": [P, I64, I64, I64, I64, I64, P, I64, I32, I32, I32, I32, P, EP, P],
    "uav_instnorm_relu": [P, I64, I64, I64, F32, I32, P, P, P],
    "uav_add_relu": [P, P, P, I64, P],
    "uav_raft_split_tanh_relu": [P, I64, I64, P, I64, P, I64, P, I64, P],
    "uav_avgpool2x2_f32": [P, I64, I64, I64, P, P],
    "uav_raft_corr_lookup": [P, P, P, P, I64, P, I64, P],
    "uav_raft_gru_rh": [P, I64, P, I64, P, I64, I64, I64, P],
    "uav_raft_gru_update": [P, I64, P, I64, P, I64, I64, I64, P],
    "uav_raft_flow_update": [P, P, I64, I64, I64, I64, P, I64, P, I64, P, I64, P],
    "uav_raft_convex_upsample": [P, P, I64, I64, I64, I64, P, P],
    "uav_attention_causal": [P, P, P, P, I64, I32, I32, I64, I64, I64, I64, I64, F32, P],
    "uav_bicubic_upsample": [P, I64, I64, I64, I32, P, P],
    "uav_plane_stats": [P, I64, I64, F32, P, P, P, P],
    "uav_adain_apply": [P, I64, I64, P, P, P, P, P, P],
    "uav_wavelet_level": [P, I64, I64, I64, I32, P, P, I32, P, P],
    "uav_pack_video_uint8": [P, I64, I64, I64, I64, P, P],
    "uav_pack_frames_png": [P, I64, I64, I64, I64, P, P],
    "uav_unpack_video_uint8": [P, I64, I64, I64, I64, I64, I32, P, P],
    "uav_rmsnorm": [P, I64, I64, I64, P, F32, P, I64, P],
    "uav_rope_kv_append": [P, I64, I64, I32, I32, I64, P, I64, P, P, I64, I64, P],
    "uav_swiglu": [P, I64, I64, I64, P, I64, P],
    "uav_gemv": [P, I64, I64, P, P, P, I32, P],
    "uav_attention_decode": [P, P, P, I64, I64, I32, I32, F32, P, P, C.c_size_t, P],
    "uav_sample_top_p": [P, I64, F32, F32, F32, P, P],
    "uav_gemv_rows": [P, I64, I64, P, I64, P, P, I32, P],
    "uav_rope_kv_append_batched": [P, I64, I64, I64, I64, I32, I32, I64, P, I64, P, P, I64, I64, I64, P],
    "uav_attention_decode_batched": [P, I64, P, P, I64, I64, I64, I64, I32, I32, F32, P, I64, P, C.c_size_t, P],
    "uav_sample_top_p_batched": [P, I64, I64, I64, F32, F32, P, P, P],
}
# include/uav_b200_int8.h: the weight-only int8 decoder Linears of the LLaVA captioner (all int status)
_INT8_PROTOS = {
    "uav_quantize_rows_int8": [P, I64, I64, I64, P, P, P],
    "uav_dequantize_rows_int8": [P, P, I64, I64, P, P],
    "uav_gemv_rows_int8": [P, P, I64, I64, P, I64, P, P, I32, P],
}
_SPECIAL = {
    "uav_version": (C.c_char_p, []),
    "uav_last_error_string": (C.c_char_p, []),
    "uav_launch_count": (C.c_uint64, []),
    "uav_groupnorm_workspace_bytes": (C.c_size_t, [I64, I32]),
    "uav_gn_partial_blocks": (C.c_int64, [I64, I64, I64]),
    "uav_plane_stats_workspace_bytes": (C.c_size_t, [I64]),
    "uav_instnorm_workspace_bytes": (C.c_size_t, [I64, I64]),
    "uav_attention_decode_workspace_bytes": (C.c_size_t, [I32, I64]),
    "uav_attention_decode_batched_workspace_bytes": (C.c_size_t, [I64, I32, I64]),
}


def lib_path() -> Path:
    return _LIB_PATH


def declared_symbols():
    """the symbols of include/uav_b200.h"""
    return list(_PROTOS) + list(_SPECIAL)


def declared_int8_symbols():
    """the symbols of include/uav_b200_int8.h"""
    return list(_INT8_PROTOS)


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise UavError(
            f"{_LIB_PATH} not found: build it with `python -m upscale_a_video_b200.build` "
            "(nvcc, sm_90a). There is no CPU / PyTorch fallback for the sampling path."
        )
    lib = C.CDLL(str(_LIB_PATH))
    for name, argtypes in (*_PROTOS.items(), *_INT8_PROTOS.items()):
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = C.c_int
    for name, (restype, argtypes) in _SPECIAL.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = restype
    _lib = lib
    return lib


def check(status: int, what: str):
    if status != 0:
        msg = load().uav_last_error_string().decode(errors="replace")
        raise UavError(f"{what} failed (status {status}): {msg}")


def launch_count() -> int:
    return int(load().uav_launch_count())
