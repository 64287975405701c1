"""ctypes binding of libsupir_b200.so (the C ABI declared in include/supir_b200.h).

There is no CPU fallback: if the library is missing, or a call is made without a CUDA device, this module raises.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsupir_b200.so")

c_void_p, c_int, c_ll, c_float, c_double = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_double


class Epilogue(ctypes.Structure):
    """struct supir_epilogue (include/supir_b200.h)."""
    _fields_ = [("bias", c_void_p), ("rowvec", c_void_p), ("rows_per_batch", c_int), ("rowvec_ld", c_int),
                ("residual", c_void_p), ("ldr", c_ll), ("act", c_int), ("out_f32", c_int), ("ln_stats", c_void_p), ("ln_colsum", c_void_p)]


class ConvGeometry(ctypes.Structure):
    """struct supir_conv_geometry (include/supir_b200.h)."""
    _fields_ = [(n, c_int) for n in ("kh", "kw", "stride", "off_y", "off_x", "Hout", "Wout", "out_sy", "out_sx", "out_oy", "out_ox",
                                     "out_H", "out_W")]


# name -> argtypes (all return int unless listed in _SPECIAL)
_SIGS = {
    "supir_gemm_bf16": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, ctypes.POINTER(Epilogue), c_void_p],
    "supir_conv3x3_bf16": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(Epilogue), c_void_p],
    "supir_conv_geom_bf16": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(ConvGeometry),
                             ctypes.POINTER(Epilogue), c_void_p],
    "supir_gemm_fp8": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, ctypes.POINTER(Epilogue),
                       c_void_p],
    "supir_conv3x3_fp8": [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_int,
                          ctypes.POINTER(Epilogue), c_void_p],
    "supir_set_gemm_tile_n": [c_int],
    "supir_conv3x3_small_cin": [c_void_p, c_ll, c_ll, c_ll, c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "supir_im2col_3x3_small_cin": [c_void_p, c_ll, c_ll, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "supir_conv3x3_small_cout": [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_ll, c_ll, c_ll, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "supir_conv1x1_small_nchw": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_float, c_void_p],
    "supir_groupnorm_stats": [c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p, c_ll, c_void_p],
    "supir_groupnorm_finalize": [c_void_p, c_int, c_double, c_void_p, c_void_p, c_void_p],
    "supir_groupnorm_merge_tiles": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "supir_groupnorm_apply": [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_void_p],
    "supir_zerosft_apply": [c_void_p, c_ll, c_void_p, c_ll, c_int, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p],
    "supir_layernorm_bf16": [c_void_p, c_ll, c_void_p, c_ll, c_ll, c_int, c_void_p, c_void_p, c_float, c_void_p],
    "supir_layernorm_stats": [c_void_p, c_ll, c_ll, c_int, c_float, c_void_p, c_void_p],
    "supir_layernorm_quant": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_int, c_void_p, c_void_p, c_float, c_void_p],
    "supir_groupnorm_apply_quant": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p, c_float, c_int, c_void_p],
    "supir_softmax_rows": [c_void_p, c_ll, c_void_p, c_ll, c_ll, c_int, c_float, c_void_p],
    "supir_attention_bf16": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p],
    "supir_attention_1head_bf16": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_float, c_void_p],
    "supir_set_attention_exp_emulation": [c_int],
    "supir_set_attention_alu_pack": [c_int],
    "supir_attention_quant_fp8": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p,
                                  c_void_p, c_ll, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "supir_attention_fp8": [c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_ll, c_int, c_int,
                            c_int, c_int, c_int, c_float, c_void_p],
    "supir_upsample_nearest2x": [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_void_p],
    "supir_im2col_3x3_s2": [c_void_p, c_ll, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "supir_copy2d_bf16": [c_void_p, c_ll, c_void_p, c_ll, c_ll, c_int, c_void_p],
    "supir_axpy_bf16": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_ll, c_int, c_void_p, c_void_p],
    "supir_nchw_f32_to_nhwc_bf16": [c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_void_p],
    "supir_nhwc_bf16_to_nchw_f32": [c_void_p, c_ll, c_void_p, c_int, c_int, c_int, c_void_p],
    "supir_nhwc_bf16_crop_to_nchw_f32": [c_void_p, c_ll, c_void_p, c_ll, c_ll, c_ll, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "supir_f32_to_bf16": [c_void_p, c_void_p, c_ll, c_void_p],
    "supir_quantize_rows": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_int, c_void_p],
    "supir_timestep_embedding": [c_void_p, c_void_p, c_int, c_int, c_void_p],
    "supir_linear_small_m": [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p],
    "supir_edm_pre": [c_void_p, c_void_p, c_float, c_float, c_void_p, c_void_p, c_ll, c_void_p],
    "supir_edm_post": [c_void_p, c_void_p, c_void_p, c_float, c_float, c_float, c_float, c_float, c_void_p, c_void_p, c_ll, c_void_p],
    "supir_axpby_f32": [c_void_p, c_float, c_void_p, c_float, c_void_p, c_ll, c_void_p],
    "supir_cfg_combine": [c_void_p, c_void_p, c_void_p, c_int, c_ll, c_void_p],
    "supir_tile_gather": [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "supir_tile_blend": [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "supir_wavelet_level": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "supir_plane_stats": [c_void_p, c_int, c_ll, c_void_p, c_ll, c_void_p],
    "supir_adain_apply": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_ll, c_void_p],
    "supir_image_to_uint8_bicubic": [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p],
    "supir_gather_rows_f32": [c_void_p, c_ll, c_int, c_void_p, c_void_p, c_ll, c_int, c_void_p, c_ll, c_ll, c_int, c_void_p],
    "supir_layernorm_f32": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_ll, c_int, c_void_p, c_void_p, c_float, c_void_p],
    "supir_attention_small_bf16": [c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p],
    "supir_activation_bf16": [c_void_p, c_ll, c_void_p, c_ll, c_ll, c_int, c_int, c_void_p],
    "supir_gaussian_latent": [c_void_p, c_void_p, c_float, c_void_p, c_int, c_int, c_ll, c_void_p],
}
# fp16 twins (include/supir_b200.h): same signature as the bf16 entry point they mirror
F16_TWINS = {
    "supir_gemm_bf16": "supir_gemm_f16", "supir_conv3x3_bf16": "supir_conv3x3_f16", "supir_conv_geom_bf16": "supir_conv_geom_f16",
    "supir_attention_bf16": "supir_attention_f16",
    "supir_groupnorm_stats": "supir_groupnorm_stats_f16", "supir_groupnorm_apply": "supir_groupnorm_apply_f16",
    "supir_zerosft_apply": "supir_zerosft_apply_f16", "supir_layernorm_bf16": "supir_layernorm_f16",
    "supir_layernorm_stats": "supir_layernorm_stats_f16",
    "supir_conv3x3_small_cin": "supir_conv3x3_small_cin_f16", "supir_im2col_3x3_small_cin": "supir_im2col_3x3_small_cin_f16",
    "supir_conv3x3_small_cout": "supir_conv3x3_small_cout_f16", "supir_nhwc_bf16_crop_to_nchw_f32": "supir_nhwc_f16_crop_to_nchw_f32",
    "supir_axpy_bf16": "supir_axpy_f16", "supir_f32_to_bf16": "supir_f32_to_f16", "supir_linear_small_m": "supir_linear_small_m_f16",
}
_SIGS.update({f16: _SIGS[bf16] for bf16, f16 in F16_TWINS.items()})

_SPECIAL = {
    "supir_last_error": ([], ctypes.c_char_p),
    "supir_version": ([], c_int),
    "supir_launch_count": ([], c_ll),
    "supir_groupnorm_stats_workspace": ([c_int, c_int, c_int, c_int], c_ll),
    "supir_plane_stats_workspace": ([c_int], c_ll),
    "supir_reset_launch_count": ([], None),
}

EXPORTED_SYMBOLS = sorted(list(_SIGS) + list(_SPECIAL))

_lib = None


class SupirNativeError(RuntimeError):
    pass


def load():
    """Load the shared library (does not need a GPU; kernels do)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SupirNativeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(make -C supir_b200/csrc). supir_b200 has no CPU or PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, args in _SIGS.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = c_int
    for name, (args, res) in _SPECIAL.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = res
    _lib = lib
    return lib


def call(name, *args):
    """Invoke an int-returning entry point; non-zero return codes become exceptions (the reference's convention)."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise SupirNativeError(f"{name} failed (rc={rc}): {lib.supir_last_error().decode(errors='replace')}")


def launch_count():
    return int(load().supir_launch_count())


def reset_launch_count():
    load().supir_reset_launch_count()
