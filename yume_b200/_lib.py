"""ctypes binding of libyume_b200.so (include/yume_b200.h). The library is mandatory: there is no Python /
PyTorch / CPU fallback for any op — a missing library is a hard error."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "csrc" / "libyume_b200.so"

YB_EPI_BF16, YB_EPI_GELU_BF16, YB_EPI_F32, YB_EPI_GATE_RES, YB_EPI_GELU_ERF_BF16, YB_EPI_RES_BF16 = 0, 1, 2, 3, 4, 5
YB_ATT_P_SMEM, YB_ATT_ACCUMULATE = 1, 2
ABI_VERSION = 4   # yb_abi_version() of the library this binding was written against
YB_ATT_EMU_SHIFT, YB_ATT_SPLIT_SHIFT = 2, 4

_ERRORS = {
    -1: "YB_ERR_ARG (null pointer / bad enum / non-positive size)",
    -2: "YB_ERR_SHAPE (shape not supported by the kernel)",
    -3: "YB_ERR_ALIGNMENT (pointer or stride not 16-byte aligned)",
    -4: "YB_ERR_NO_DRIVER (cuTensorMapEncodeTiled unavailable: no CUDA driver)",
    -5: "YB_ERR_TENSORMAP (driver rejected a TMA descriptor)",
    -6: "YB_ERR_LAUNCH (kernel launch failed)",
}


class YumeB200Error(RuntimeError):
    pass


class GemmArgs(C.Structure):
    """Mirror of `struct yb_gemm_args` (include/yume_b200.h)."""

    _fields_ = [
        ("struct_bytes", C.c_uint), ("cta_pair", C.c_int),
        ("A", C.c_void_p), ("B", C.c_void_p), ("bias", C.c_void_p), ("out", C.c_void_p),
        ("gate", C.c_void_p), ("tok_idx", C.c_void_p),
        ("lda", C.c_longlong), ("ldb", C.c_longlong), ("ldo", C.c_longlong), ("gate_ld", C.c_longlong),
        ("M", C.c_int), ("N", C.c_int), ("K", C.c_int), ("epilogue", C.c_int), ("block_n", C.c_int),
        ("n_split", C.c_int), ("split_stride", C.c_longlong), ("a_split", C.c_int), ("a_split_stride", C.c_longlong),
        ("res", C.c_void_p), ("res_ld", C.c_longlong),
        ("split_k", C.c_int), ("ws", C.c_void_p), ("ws_bytes", C.c_longlong),
    ]


class Conv3dArgs(C.Structure):
    """Mirror of `struct yb_conv3d_args`."""

    _fields_ = [
        ("struct_bytes", C.c_uint), ("cta_pair", C.c_int),
        ("xpad", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("out", C.c_void_p), ("res", C.c_void_p),
        ("ldo", C.c_longlong), ("res_ld", C.c_longlong),
        ("T", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cp", C.c_int), ("Cout", C.c_int), ("epilogue", C.c_int),
        ("kt", C.c_int), ("kh", C.c_int), ("kw", C.c_int), ("oob_zero_pad", C.c_int), ("out_t_mul", C.c_int),
        ("out_t_add", C.c_int), ("fuse_w", C.c_int), ("stride_t", C.c_int), ("stride_hw", C.c_int),
    ]


# name -> (restype, argtypes); every symbol include/yume_b200.h declares
_vp, _ll, _i, _f = C.c_void_p, C.c_longlong, C.c_int, C.c_float
SIGNATURES = {
    "yb_abi_version": (_i, []),
    "yb_gemm_bf16": (_i, [C.POINTER(GemmArgs), _vp]),
    "yb_conv3d_causal": (_i, [C.POINTER(Conv3dArgs), _vp]),
    "yb_gn_stats": (_i, [_vp, _ll, _vp, _ll, _i, _i, _vp]),
    "yb_vae_pad_act": (_i, [_vp, _ll, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i, _f, _i, _vp]),
    "yb_masked_softmax": (_i, [_vp, _ll, _vp, _ll, _i, _i, _vp]),
    "yb_nchw_to_nhwc_bf16": (_i, [_vp, _vp, _ll, _i, _i, _vp]),
    "yb_nhwc_to_nchw_f32": (_i, [_vp, _ll, _vp, _ll, _i, _vp]),
    "yb_gemm_plan": (_i, [_i, _i, _i, C.POINTER(C.c_int)]),
    "yb_gemm_workspace_bytes": (_ll, [_i, _i, _i, _i, _i, _i]),
    "yb_gemm_splitk_plan": (_i, [_i, _i, _i, _i, C.POINTER(C.c_int)]),
    "yb_conv3d_plan": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(C.c_int)]),
    "yb_attention_plan": (_i, [_i, _i, _i, _i, _i, C.POINTER(C.c_int)]),
    "yb_nhwc_to_nchw_f32_clamp": (_i, [_vp, _ll, _vp, _ll, _i, C.c_float, C.c_float, _vp]),
    "yb_blend": (_i, [_vp, _vp, _ll, _i, _i, _i, _ll, _vp]),
    "yb_vae_assemble_tiles": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp]),
    "yb_vae_rms_act": (_i, [_vp, _ll, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "yb_vae_dupup_add": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "yb_vae_unpatchify2_clamp": (_i, [_vp, _ll, _vp, _i, _i, _i, _vp]),
    "yb_vae_avgdown_add": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "yb_vae_patchify2_bf16": (_i, [_vp, _vp, _ll, _i, _i, _i, _vp]),
    "yb_ln_modulate": (_i, [_vp, _ll, _vp, _ll, _i, _vp, _vp, _ll, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "yb_rmsnorm_rope": (_i, [_vp, _ll, _vp, _vp, _i, _i, _i, _i, _f, _vp]),
    "yb_rmsnorm_rope_pieces": (_i, [_vp, _ll, _i, _ll, _vp, _vp, _i, _i, _i, _i, _f, _vp]),
    "yb_qk_norm_rope": (_i, [_vp, _vp, _ll, _i, _ll, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp]),
    "yb_attention": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _ll, _i, _i, _i, _f, _i, _vp]),
    "yb_attention_ex": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _ll, _i, _i, _i, _f, _i, _vp, _ll, _vp, _vp]),
    "yb_attention_workspace_bytes": (_ll, [_i, _i, _i, _i, _i]),
    "yb_debug_force_split": (_i, [_i]),
    "yb_sp_scatter_qkv": (_i, [_vp, _ll, _vp, _vp, _vp, _i, _i, _i, _i, _f, C.POINTER(C.c_void_p), _i, _i, _i, _vp]),
    "yb_gemm_sp_qkv": (_i, [_vp, _ll, _vp, _vp, _i, _i, _i, C.POINTER(C.c_void_p), _i, _i, _i, _vp, _vp]),
    "yb_sp_bcast_sums": (_i, [_vp, C.POINTER(C.c_void_p), _i, _i, _i, _vp]),
    "yb_sp_post_norm_rope": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp]),
    "yb_attention_sp": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, C.POINTER(C.c_void_p), _ll, _i, _i, _i, _f, _i, _i, _i, _i, _vp, _ll,
                             _vp]),
    "yb_patchify": (_i, [_vp, _ll, _ll, _ll, _ll, _vp, _ll, _i, _i, _i, _i, _i, _i, _vp]),
    "yb_bcast_add": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp]),
    "yb_unpatchify": (_i, [_vp, _ll, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "yb_sinusoidal": (_i, [_vp, _vp, _i, _i, _vp]),
    "yb_linear_f32_small": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "yb_linear_f32": (_i, [_vp, _ll, _vp, _vp, _vp, _ll, _i, _i, _i, _vp]),
    "yb_umma_probe": (_i, [_vp, _vp, _vp, _i, _vp]),
}

# every symbol include/yume_b200_clip.h declares (the CLIP vision encoder's input kernel)
CLIP_SIGNATURES = {
    "yb_resize_bicubic_normalize": (_i, [_vp, _ll, _ll, _ll, _i, _i, _i, _vp, _i, _vp, _vp, _vp]),
}

# every symbol include/yume_b200_t5.h declares (the umT5 text encoder's attention, RMS norm and gated GELU)
T5_SIGNATURES = {
    "yb_t5_attention": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _ll, _i, _i, _i, _vp, _vp, _vp]),
    "yb_t5_rmsnorm": (_i, [_vp, _ll, _vp, _ll, _i, _vp, _i, _i, _f, _vp]),
    "yb_t5_geglu": (_i, [_vp, _ll, _vp, _ll, _i, _i, _vp]),
}

# every symbol include/yume_b200_stream.h declares (the chunk-streaming forms of the Wan VAE kernels)
STREAM_SIGNATURES = {
    "yb_conv3d_causal_hist": (_i, [C.POINTER(Conv3dArgs), _i, _vp]),
    "yb_vae_dupup_add_cont": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "yb_vae_unpatchify2_clamp_win": (_i, [_vp, _ll, _vp, _ll, _i, _i, _i, _vp]),
    "yb_nhwc_to_nchw_f32_clamp_win": (_i, [_vp, _ll, _vp, _ll, _ll, _i, _f, _f, _vp]),
    "yb_vae_patchify2_bf16_win": (_i, [_vp, _ll, _vp, _ll, _i, _i, _i, _vp]),
    "yb_nchw_to_nhwc_bf16_win": (_i, [_vp, _ll, _vp, _ll, _i, _i, _vp]),
}

# every symbol include/yume_b200_fp8.h declares (the opt-in FP8 block GEMMs and their activation quantisers)
YB_EPI_GELU_FP8 = 8


class GemmFp8Args(C.Structure):
    """Mirror of `struct yb_gemm_fp8_args` (include/yume_b200_fp8.h)."""

    _fields_ = [
        ("struct_bytes", C.c_uint), ("M", C.c_int), ("N", C.c_int), ("K", C.c_int),
        ("A", C.c_void_p), ("a_scale", C.c_void_p), ("B", C.c_void_p), ("b_scale", C.c_void_p), ("bias", C.c_void_p),
        ("out", C.c_void_p), ("out_scale", C.c_void_p), ("gate", C.c_void_p), ("tok_idx", C.c_void_p),
        ("lda", C.c_longlong), ("lds", C.c_longlong), ("ldb", C.c_longlong), ("ldo", C.c_longlong), ("ldos", C.c_longlong),
        ("gate_ld", C.c_longlong), ("epilogue", C.c_int), ("block_n", C.c_int),
    ]


FP8_SIGNATURES = {
    "yb_gemm_fp8": (_i, [C.POINTER(GemmFp8Args), _vp]),
    "yb_ln_modulate_fp8": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _vp, _ll, _vp, _vp, _vp, _i, _i, _f, _vp]),
    "yb_quant_rows_fp8": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _i, _i, _vp]),
}

# every symbol include/yume_b200_fp8_attn.h declares (the e4m3 self-attention of precision="fp8_attn")
FP8_ATTN_SIGNATURES = {
    "yb_quant_vt_fp8": (_i, [_vp, _ll, _vp, _vp, _i, _i, _vp]),
    "yb_attention_fp8": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _vp, _vp, _ll, _i, _i, _i, _f, _i, _vp, _ll, _vp]),
}

# every symbol include/yume_b200_fp8_sp.h declares (precision="fp8" / "fp8_attn" under Ulysses sequence parallelism)
FP8_SP_SIGNATURES = {
    "yb_quant_rows_fp8_split": (_i, [_vp, _ll, _i, _ll, _vp, _ll, _vp, _ll, _i, _i, _vp]),
    "yb_attention_fp8_sp": (_i, [_vp, _ll, _vp, _ll, _vp, _ll, _vp, _vp, C.POINTER(C.c_void_p), _ll, _i, _i, _i, _f, _i, _i, _i,
                                 _i, _vp, _ll, _vp]),
    "yb_sp_pack_qkv": (_i, [_vp, _ll, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _i, _i, _vp]),
}

# every symbol include/yume_b200_fp8_vae.h declares (the e4m3 convs of Wan22VaeDecoder(precision="fp8"))
class Conv3dFp8Args(C.Structure):
    """Mirror of `struct yb_conv3d_fp8_args` (include/yume_b200_fp8_vae.h)."""

    _fields_ = [
        ("struct_bytes", C.c_uint), ("x", C.c_void_p), ("x_scale", C.c_void_p), ("w", C.c_void_p), ("w_scale", C.c_void_p),
        ("bias", C.c_void_p), ("out", C.c_void_p), ("res", C.c_void_p), ("ldo", C.c_longlong), ("res_ld", C.c_longlong),
        ("T", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cp", C.c_int), ("Cout", C.c_int),
        ("kt", C.c_int), ("kh", C.c_int), ("kw", C.c_int), ("t_hist", C.c_int), ("epilogue", C.c_int),
    ]


FP8_VAE_SIGNATURES = {
    "yb_conv3d_fp8": (_i, [C.POINTER(Conv3dFp8Args), _vp]),
    "yb_vae_rms_act_fp8": (_i, [_vp, _ll, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
}

# every symbol include/yume_b200_vae_resume.h declares (the frame comparison of a resuming Wan VAE session)
RESUME_SIGNATURES = {
    "yb_vae_frame_match": (_i, [_vp, _i, _vp, _i, _i, _ll, _i, _vp, _vp]),
}

# every symbol include/yume_b200_vae_rows.h declares (the row-band forms of a row-parallel Wan VAE decode)
ROWS_SIGNATURES = {
    "yb_conv3d_rows": (_i, [C.POINTER(Conv3dArgs), _i, _vp]),
    "yb_vae_rms_act_rows": (_i, [_vp, _ll, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "yb_vae_rows_pack": (_i, [_vp, _vp, _i, _i, _ll, _vp]),
    "yb_vae_rows_unpack": (_i, [_vp, _vp, _vp, _i, _i, _ll, _vp]),
    "yb_vae_unpatchify2_clamp_rows": (_i, [_vp, _ll, _vp, _ll, _ll, _i, _i, _i, _vp]),
    "yb_nhwc_to_nchw_f32_clamp_rows": (_i, [_vp, _ll, _vp, _ll, _ll, _i, _i, _i, _i, _f, _f, _vp]),
}

# every symbol include/yume_b200_vae_rows_enc.h declares (the row-band forms of a row-parallel Wan VAE encode)
ROWS_ENC_SIGNATURES = {
    "yb_conv3d_rows_down": (_i, [C.POINTER(Conv3dArgs), _vp]),
    "yb_vae_patchify2_bf16_rows": (_i, [_vp, _ll, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "yb_nchw_to_nhwc_bf16_rows": (_i, [_vp, _ll, _vp, _i, _i, _i, _i, _i, _i, _i, _vp]),
}

_lib = None


def lib_path() -> Path:
    return _LIB_PATH


def load():
    """Load the shared library (once). Raises YumeB200Error if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise YumeB200Error(
            f"{_LIB_PATH} is missing: build it with `python -m yume_b200.build` (or __graft_entry__.build()). "
            "yume_b200 has no fallback path.")
    lib = C.CDLL(str(_LIB_PATH))
    if lib.yb_abi_version() != ABI_VERSION:
        raise YumeB200Error(f"{_LIB_PATH} has ABI version {lib.yb_abi_version()}, this binding expects {ABI_VERSION}: rebuild it "
                            "(python -m yume_b200.build --force)")
    for name, (res, args) in {**SIGNATURES, **CLIP_SIGNATURES, **T5_SIGNATURES, **STREAM_SIGNATURES,
                              **FP8_SIGNATURES, **FP8_ATTN_SIGNATURES, **FP8_VAE_SIGNATURES, **RESUME_SIGNATURES,
                              **FP8_SP_SIGNATURES, **ROWS_SIGNATURES, **ROWS_ENC_SIGNATURES}.items():
        fn = getattr(lib, name)  # AttributeError here means header and library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise YumeB200Error(f"{what} failed: {_ERRORS.get(rc, rc)}")
